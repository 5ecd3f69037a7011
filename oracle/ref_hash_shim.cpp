// oracle/_ref: the REAL hash functions of the exchange / join path, compiled from the reference tree where they lie:
//   HashUtil::fnv_hash, HashUtil::zlib_crc_hash  (be/src/base/hash/hash_util.hpp:34-45,127-134: the ExchangeSink partition
//     hashes of column_hash.cpp / exchange_sink_operator.cpp:586-637),
//   crc_hash_32  (be/src/base/hash/hash.h:96-130: JoinKeyHash<Slice> and the 1/2-byte JoinKeyHash, join_hash_map_helper.h:27,60).
// be/src/base/hash/hash_util.cpp and be/src/gutil/cpu.cc are compiled along for the out-of-line parts; oracle/ref_shims/ stands
// in for glog / butil.  Built by `make -C oracle ref` only where a reference tree is given; tests/test_oracle_golden.py checks the
// restatements (orc_fnv_hash, orc_zlib_crc32, orc_crc_hash_32) against it on random byte strings.
#include "base/hash/hash.h"
#include "base/hash/hash_util.hpp"

using namespace starrocks;

extern "C" unsigned ref_fnv_hash(const void* d, int n, unsigned seed) { return HashUtil::fnv_hash(d, n, seed); }
extern "C" unsigned ref_zlib_crc_hash(const void* d, int n, unsigned seed) { return HashUtil::zlib_crc_hash(d, n, seed); }
extern "C" unsigned ref_crc_hash_32(const void* d, int n, unsigned seed) { return crc_hash_32(d, n, seed); }

// referenced by HashUtil::murmur_hash3_128 only (not on this path): never called here
void murmur_hash3_x64_64(const void*, int, uint64_t, void*) { __builtin_trap(); }
