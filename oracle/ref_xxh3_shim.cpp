// oracle/_ref: the REAL reference code for the one piece of the path that compiles from the reference tree on its own --
// the vendored single-header xxHash (be/src/base/hash/xxhash.h) behind HashUtil::xx_hash3_64
// (be/src/base/hash/hash_util.cpp:100-102).  Built by `make -C oracle ref` ONLY where a reference tree is given; the header is
// included from where it lies (no reference source is copied into this repository); the output goes to oracle/_ref/.
// tests/test_oracle_golden.py cross-checks orc_xxh3_64 (the restatement) against it on random inputs.
#ifndef SR_REFERENCE_XXHASH
#error "define SR_REFERENCE_XXHASH to the path of the reference's be/src/base/hash/xxhash.h"
#endif
#define XXH_INLINE_ALL
#include SR_REFERENCE_XXHASH

extern "C" unsigned long long ref_xx_hash3_64(const void* key, int len, unsigned long long seed) { return XXH3_64bits_withSeed(key, (size_t)len, seed); }
