// Scratch measurement (not part of the product): cost of sparse 4-byte reads of pinned host memory from a kernel.
//  (1) as a function of the distance between the words read -> the PCIe read granularity a late-materialising pass
//      pays per surviving row (kernel reads of mapped host memory move 64-byte blocks);
//  (2) the same number of sparse reads spread over 1 or 4 separate columns, independent or chained, grid-stride or
//      block-contiguous -> how a gather pass should be organised.
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o pcie_stride pcie_stride.cu
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

__global__ void k_stride(const int* __restrict__ p, int64_t nwords, int stride_words, int per_thread, unsigned long long* out) {
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t nth = (int64_t)gridDim.x * blockDim.x;
    int acc = 0;
    for (int64_t k = tid; k * stride_words < nwords; k += nth * per_thread) {
#pragma unroll 8
        for (int u = 0; u < per_thread; u++) {
            const int64_t w = (k + (int64_t)u * nth) * stride_words;
            if (w < nwords) acc ^= __ldg(p + w);
        }
    }
    if (acc == 0x7fffffff) atomicAdd(out, 1ull);
}

// NC columns of `colwords` words each; row r of column c is p[c*colwords + r]; rows visited: every `stride_words`-th
// (+ a per-row jitter so that rows are not perfectly regular).  chained: the address of column c+1 depends on the
// value read from column c (value == row index by construction, so the address is the same).
template <int NC, bool CHAINED, bool BLOCK_CONTIG>
__global__ void k_cols(const int* __restrict__ p, int64_t colwords, int stride_words, unsigned long long* out) {
    const int64_t nrows = colwords / stride_words;
    const int64_t nth = (int64_t)gridDim.x * blockDim.x;
    int acc = 0;
    int64_t k, kend, kstep;
    if (BLOCK_CONTIG) {
        const int64_t per_block = (nrows + gridDim.x - 1) / gridDim.x;
        k = (int64_t)blockIdx.x * per_block + threadIdx.x;
        kend = min(nrows, ((int64_t)blockIdx.x + 1) * per_block);
        kstep = blockDim.x;
    } else {
        k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
        kend = nrows;
        kstep = nth;
    }
    for (; k < kend; k += kstep) {
        int64_t r = k * stride_words + (k * 2654435761u >> 7) % stride_words;
#pragma unroll
        for (int c = 0; c < NC; c++) {
            const int v = __ldg(p + (int64_t)c * colwords + r);
            acc ^= v;
            if (CHAINED) r = v;
        }
    }
    if (acc == 0x7fffffff) atomicAdd(out, 1ull);
}

template <typename F>
static float best_of(F launch) {
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    float best = 1e9f;
    for (int rep = 0; rep < 3; rep++) {
        cudaEventRecord(e0);
        launch();
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        float ms;
        cudaEventElapsedTime(&ms, e0, e1);
        if (ms < best) best = ms;
    }
    return best;
}

int main() {
    const int64_t bytes = 8ll << 30;
    const int64_t colwords = bytes / 4 / 4; // 4 columns of 2 GiB
    int* h;
    if (cudaHostAlloc(&h, bytes, cudaHostAllocMapped) != cudaSuccess) {
        printf("host alloc failed\n");
        return 1;
    }
    for (int c = 0; c < 4; c++)
        for (int64_t i = 0; i < colwords; i++) h[c * colwords + i] = (int)i;
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    unsigned long long* out;
    cudaMalloc(&out, 8);
    cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, 32);
    const int strides[] = {1, 8, 16, 32, 64, 256};
    for (int s : strides) {
        const float ms = best_of([&] { k_stride<<<sms * 8, 256>>>(h, colwords, s, 4, out); });
        const double reqs = (double)colwords / s;
        printf("1 column, stride %4d B: %8.2f ms  %7.1f M words/s\n", s * 4, ms, reqs / ms / 1e3);
    }
    for (int s : {16, 64}) { // rows 64 B / 256 B apart
        const double reqs1 = (double)(colwords / s);
        float ms;
        ms = best_of([&] { k_cols<1, false, false><<<sms * 4, 256>>>(h, colwords, s, out); });
        printf("stride %4d B  1 col               grid-stride: %8.2f ms %7.1f M reads/s\n", s * 4, ms, reqs1 / ms / 1e3);
        ms = best_of([&] { k_cols<4, false, false><<<sms * 4, 256>>>(h, colwords, s, out); });
        printf("stride %4d B  4 cols independent  grid-stride: %8.2f ms %7.1f M reads/s\n", s * 4, ms, 4 * reqs1 / ms / 1e3);
        ms = best_of([&] { k_cols<4, true, false><<<sms * 4, 256>>>(h, colwords, s, out); });
        printf("stride %4d B  4 cols chained      grid-stride: %8.2f ms %7.1f M reads/s\n", s * 4, ms, 4 * reqs1 / ms / 1e3);
        ms = best_of([&] { k_cols<1, false, true><<<sms * 4, 256>>>(h, colwords, s, out); });
        printf("stride %4d B  1 col               block-contig: %8.2f ms %7.1f M reads/s\n", s * 4, ms, reqs1 / ms / 1e3);
        ms = best_of([&] { k_cols<4, false, true><<<sms * 4, 256>>>(h, colwords, s, out); });
        printf("stride %4d B  4 cols independent  block-contig: %8.2f ms %7.1f M reads/s\n", s * 4, ms, 4 * reqs1 / ms / 1e3);
        ms = best_of([&] { k_cols<4, true, true><<<sms * 4, 256>>>(h, colwords, s, out); });
        printf("stride %4d B  4 cols chained      block-contig: %8.2f ms %7.1f M reads/s\n", s * 4, ms, 4 * reqs1 / ms / 1e3);
    }
    printf("%s\n", cudaGetErrorString(cudaGetLastError()));
    return 0;
}
