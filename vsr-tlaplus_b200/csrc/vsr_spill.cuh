/*
 * vsr_spill.cuh — a buffer of fixed-size rows that continues in pinned host memory, mapped into the device, once its part in
 * HBM is full (BASELINE configs[3]): the two frontier buffers, the liveness store's words and the trace.  Row i is at hbm + i * NW while
 * i < split, and at host + (i - split) * NW after that.  Without a host part split = ~0, so "does this lie in HBM" is one
 * compare on the hot path.
 */
#ifndef VSR_SPILL_CUH
#define VSR_SPILL_CUH

#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

namespace vsr {

/* TMA bulk store shared -> global of `bytes` (multiple of 16), issued by one lane; waits until the
   shared source may be overwritten */
__device__ __forceinline__ void bulk_store(void* gdst, const void* ssrc, uint32_t bytes) {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    const uint32_t s = (uint32_t)__cvta_generic_to_shared(ssrc);
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(s), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}

/* what a kernel gets: the rows of one spilled buffer, by value inside its parameter struct */
struct SpillRows {
    uint32_t* hbm;
    uint32_t* host;           /* NULL without a host part */
    unsigned long long split; /* rows in the HBM part; ~0 without a host part */

    template <int NW> __host__ __device__ __forceinline__ uint32_t* row(unsigned long long i) const {
        return i < split ? hbm + i * NW : host + (i - split) * NW;
    }
    /* rows [first, first + n) all lie in the HBM part */
    __host__ __device__ __forceinline__ bool in_hbm(unsigned long long first, unsigned long long n) const { return first + n <= split; }
    /* the rows from row `first` on, as a view whose row 0 is that row */
    SpillRows from(unsigned long long first, int nw) const {
        if (first < split) return {hbm + first * nw, host, split == ~0ull ? ~0ull : split - first};
        return {host + (first - split) * nw, nullptr, ~0ull};
    }
};

/* n (<= 32) rows of NW words staged in shared memory, stored to rows [base, base + n): one bulk store, or two when the
   rows straddle the end of the HBM part */
template <int NW> __device__ __forceinline__ void store_rows(const SpillRows& r, unsigned long long base, const uint32_t* stage, int n) {
    if (base + n <= r.split) bulk_store(r.hbm + base * NW, stage, (uint32_t)(n * NW * 4));
    else if (base >= r.split) bulk_store(r.host + (base - r.split) * NW, stage, (uint32_t)(n * NW * 4));
    else {
        const int n1 = (int)(r.split - base);
        bulk_store(r.hbm + base * NW, stage, (uint32_t)(n1 * NW * 4));
        bulk_store(r.host, stage + n1 * NW, (uint32_t)((n - n1) * NW * 4));
    }
}

/* the host side: owns both parts of one buffer.  The caller sizes them; a part of 0 rows is not allocated. */
struct SpillBuffer {
    uint32_t* hbm = nullptr;
    uint32_t* host = nullptr;
    uint64_t hbm_rows = 0, host_rows = 0, row_bytes = 0;

    /* the HBM part, on `st` (the engine's stream and memory pool) */
    cudaError_t alloc_hbm(uint64_t rows, uint64_t bytes_per_row, cudaStream_t st) {
        hbm_rows = rows;
        row_bytes = bytes_per_row;
        return rows ? cudaMallocAsync((void**)&hbm, rows * row_bytes, st) : cudaSuccess;
    }
    /* the host part: pinned, device-mapped, usable from every device */
    cudaError_t alloc_host(uint64_t rows) {
        host_rows = rows;
        return rows ? cudaHostAlloc((void**)&host, rows * row_bytes, cudaHostAllocPortable | cudaHostAllocMapped) : cudaSuccess;
    }
    /* no kernel may still use the host part when it is freed: the stream is synchronised first */
    void release(cudaStream_t st) {
        if (st) { cudaFreeAsync(hbm, st); cudaStreamSynchronize(st); }
        else cudaFree(hbm);
        if (host) cudaFreeHost(host);
        hbm = host = nullptr;
    }
    uint64_t capacity() const { return hbm_rows + host_rows; }
    SpillRows view() const { return {hbm, host, host_rows ? hbm_rows : ~0ull}; }
    /* the same memory as rows of `words` 4-byte words (scratch space for another kind of row), and how many fit */
    SpillRows view_as(int words) const { return {hbm, host, host_rows ? hbm_rows * row_bytes / (4 * words) : ~0ull}; }
    uint64_t capacity_as(int words) const { return (hbm_rows * row_bytes) / (4 * words) + (host_rows * row_bytes) / (4 * words); }
    /* rows [first, first + n) <-> host memory: the HBM part by cudaMemcpy, the host part directly */
    cudaError_t to_host(uint64_t first, uint64_t n, void* dst) const {
        const uint64_t k = first < hbm_rows ? (n < hbm_rows - first ? n : hbm_rows - first) : 0;
        const cudaError_t ce = k ? cudaMemcpy(dst, (const uint8_t*)hbm + first * row_bytes, k * row_bytes, cudaMemcpyDeviceToHost) : cudaSuccess;
        if (ce != cudaSuccess) return ce;
        if (n > k) memcpy((uint8_t*)dst + k * row_bytes, (const uint8_t*)host + (first + k - hbm_rows) * row_bytes, (n - k) * row_bytes);
        return cudaSuccess;
    }
    cudaError_t from_host(uint64_t first, uint64_t n, const void* src) {
        const uint64_t k = first < hbm_rows ? (n < hbm_rows - first ? n : hbm_rows - first) : 0;
        const cudaError_t ce = k ? cudaMemcpy((uint8_t*)hbm + first * row_bytes, src, k * row_bytes, cudaMemcpyHostToDevice) : cudaSuccess;
        if (ce != cudaSuccess) return ce;
        if (n > k) memcpy((uint8_t*)host + (first + k - hbm_rows) * row_bytes, (const uint8_t*)src + k * row_bytes, (n - k) * row_bytes);
        return cudaSuccess;
    }
};

} // namespace vsr
#endif
