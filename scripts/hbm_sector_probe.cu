// Scratch measurement (not part of the product): what HBM charges for sparse reads of one 2.4 GB int32 fact column
// (600 M rows, the SF100 lineorder column), i.e. at which granularity the fragment passes pay for the rows they touch.
//  (1) a full 128-bit streaming read (the stream pass);
//  (2) every other 32-byte sector, one sector in four, and a random 83 % of the sectors (the sectors a 20 %-dense
//      second column touches: 1 - 0.8^8) -- each sector read whole by one thread (two 128-bit loads);
//  (3) single 4-byte gathers of random rows at 1.6 % and 4 % density (the final pass and the gather-join pass).
// If reading half the sectors costs about as much as reading all of them, HBM moves 64 bytes or more per access and
// skipping single 32-byte sectors saves nothing.
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o hbm_sector_probe hbm_sector_probe.cu
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

__device__ __forceinline__ uint32_t mix(uint64_t x) {
    x ^= x >> 33;
    x *= 0xff51afd7ed558ccdull;
    x ^= x >> 33;
    x *= 0xc4ceb9fe1a85ec53ull;
    return (uint32_t)(x >> 40); // 24 bits
}

__device__ __forceinline__ int4 ld_v4(const void* p) {
    int4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ int ld_s32(const void* p) {
    int r;
    asm volatile("ld.global.nc.L1::no_allocate.s32 %0, [%1];" : "=r"(r) : "l"(p));
    return r;
}

// (1) every 16-byte chunk, grid-stride, four loads in flight per thread
__global__ void k_full(const int4* __restrict__ p, int64_t n16, unsigned long long* out) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    int acc = 0;
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (; i + 3 * stride < n16; i += 4 * stride) {
        const int4 a = ld_v4(p + i), b = ld_v4(p + i + stride), c = ld_v4(p + i + 2 * stride), d = ld_v4(p + i + 3 * stride);
        acc ^= a.x ^ b.y ^ c.z ^ d.w;
    }
    for (; i < n16; i += stride) acc ^= ld_v4(p + i).x;
    if (acc == 0x7fffffff) atomicAdd(out, 1ull);
}

// (2) one thread per 32-byte sector: sector s is read when (every > 0) s % every == 0, else (every == 0) when its hash
// falls below `keep` (of 2^24).  Four sectors per thread and iteration, so the loads of a thread overlap.
__global__ void k_sectors(const int4* __restrict__ p, int64_t nsec, int every, uint32_t keep, unsigned long long* out) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    int acc = 0;
    for (int64_t s0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s0 < nsec; s0 += 4 * stride) {
        int4 v[8];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int64_t s = s0 + u * stride;
            const bool take = s < nsec && (every > 0 ? s % every == 0 : mix((uint64_t)s) < keep);
            v[2 * u] = v[2 * u + 1] = make_int4(0, 0, 0, 0);
            if (take) {
                v[2 * u] = ld_v4(p + 2 * s);
                v[2 * u + 1] = ld_v4(p + 2 * s + 1);
            }
        }
#pragma unroll
        for (int u = 0; u < 8; u++) acc ^= v[u].x ^ v[u].w;
    }
    if (acc == 0x7fffffff) atomicAdd(out, 1ull);
}

// (3) one thread per sector, a predicated 4-byte load for each of its 8 rows whose hash falls below `keep`
__global__ void k_rows(const int* __restrict__ p, int64_t nsec, uint32_t keep, unsigned long long* out, unsigned long long* touched) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    int acc = 0;
    unsigned long long t = 0;
    for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < nsec; s += stride) {
        bool any = false;
#pragma unroll
        for (int r = 0; r < 8; r++) {
            const int64_t row = s * 8 + r;
            if (mix((uint64_t)row * 0x9E3779B97F4A7C15ull) < keep) {
                acc ^= ld_s32(p + row);
                any = true;
            }
        }
        t += any;
    }
    if (acc == 0x7fffffff) atomicAdd(out, 1ull);
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if ((threadIdx.x & 31) == 0) atomicAdd(touched, t);
}

template <typename F>
static float best_of(F launch) {
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    launch(); // warm-up
    float best = 1e9f;
    for (int rep = 0; rep < 5; rep++) {
        cudaEventRecord(e0);
        launch();
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        float ms;
        cudaEventElapsedTime(&ms, e0, e1);
        if (ms < best) best = ms;
    }
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    return best;
}

int main() {
    const int64_t rows = 600000000ll; // 2.4 GB of int32
    const int64_t bytes = rows * 4;
    const int64_t nsec = bytes / 32;
    int* d;
    if (cudaMalloc(&d, bytes) != cudaSuccess) {
        printf("device alloc failed\n");
        return 1;
    }
    cudaMemset(d, 0x5a, bytes);
    unsigned long long *out, *touched;
    cudaMalloc(&out, 8);
    cudaMalloc(&touched, 8);
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, 0);
    size_t gran = 0;
    cudaDeviceGetLimit(&gran, cudaLimitMaxL2FetchGranularity);
    printf("device: %s, %d SMs, L2 %d MB, max L2 fetch granularity %zu B (default, not changed)\n", prop.name, sms, prop.l2CacheSize >> 20, gran);
    printf("%-36s %9s %12s %10s %14s\n", "pattern", "ms", "sectors", "frac_all", "G sectors/s");
    const float full = best_of([&] { k_full<<<sms * 8, 256>>>((const int4*)d, bytes / 16, out); });
    printf("%-36s %9.3f %12lld %10.3f %14.2f   (%.0f GB/s)\n", "full 128-bit stream", full, (long long)nsec, 1.0, nsec / full / 1e6, bytes / full / 1e6);
    struct Pat {
        const char* name;
        int every;
        double keep;
    } pats[] = {{"every other 32 B sector", 2, 0}, {"one 32 B sector in four", 4, 0}, {"random 83 % of the sectors", 0, 0.83}, {"random 50 % of the sectors", 0, 0.50}};
    for (const Pat& pt : pats) {
        const uint32_t keep = (uint32_t)(pt.keep * (1u << 24));
        const float ms = best_of([&] { k_sectors<<<sms * 8, 256>>>((const int4*)d, nsec, pt.every, keep, out); });
        const double sec = pt.every > 0 ? (double)nsec / pt.every : (double)nsec * pt.keep;
        printf("%-36s %9.3f %12.0f %10.3f %14.2f   (time / full %.3f)\n", pt.name, ms, sec, sec / nsec, sec / ms / 1e6, ms / full);
    }
    for (double dens : {0.016, 0.04, 0.20}) {
        const uint32_t keep = (uint32_t)(dens * (1u << 24));
        cudaMemset(touched, 0, 8);
        k_rows<<<sms * 8, 256>>>(d, nsec, keep, out, touched);
        unsigned long long t = 0;
        cudaMemcpy(&t, touched, 8, cudaMemcpyDeviceToHost);
        const float ms = best_of([&] { k_rows<<<sms * 8, 256>>>(d, nsec, keep, out, touched); });
        char name[64];
        snprintf(name, sizeof name, "row gathers at %.1f %% density", dens * 100);
        printf("%-36s %9.3f %12llu %10.3f %14.2f   (time / full %.3f, %.1f M rows)\n", name, ms, t, (double)t / nsec, t / ms / 1e6, ms / full, rows * dens / 1e6);
    }
    printf("%s\n", cudaGetErrorString(cudaGetLastError()));
    cudaFree(d);
    return 0;
}
