/*
 * vsr_gpu_thunks.cuh — internal: the kernel launchers (GpuOps) of one compile-time Layout<R,V,K>.  Instantiated for
 * every built-in layout in vsr_gpu.cu and for one layout in a layout plug-in (vsr_layout_plugin.cu).
 */
#ifndef VSR_GPU_THUNKS_CUH
#define VSR_GPU_THUNKS_CUH

#include "vsr_gpu.cuh"
#include "vsr_live.cuh"
#include "vsr_model.h"

namespace vsr {

struct GpuOps {
    uint32_t (*check_hash)(const uint32_t*, int use_view);
    int R, V, K, nw, bytes, rec_bytes;
    size_t expand_smem;
    int states_per_block;
    cudaError_t (*launch_expand)(const ExpandParams&, int grid, cudaStream_t);
    cudaError_t (*launch_patch)(const ExpandParams&, const uint8_t* ties, unsigned long long ntie, unsigned long long n_out, cudaStream_t);
    int tie_bytes;
    cudaError_t (*prepare)(int* blocks_per_sm);
    cudaError_t (*launch_simulate)(const SimParams&, int grid, cudaStream_t);
    /* the expand kernel's shape (ExpandCfg): warps per block, blocks per SM, scan passes per round, staging rows per warp */
    int warps, blocks, passes, stage_rows;
    cudaError_t (*launch_audit)(const ExpandParams&, unsigned long long n_states, AuditSums* out, int sms, cudaStream_t);
    /* liveness pass (vsr_live.cuh): store a level's not-P states; one elimination sweep over store indices [first, first + n) */
    cudaError_t (*launch_live_collect)(const LiveParams&, int sms, cudaStream_t);
    cudaError_t (*launch_live_sweep)(const LiveParams&, int sms, cudaStream_t);
};

/* what a layout plug-in must have been compiled against: the version constant AND the shapes of the structs the kernels and the
   host exchange (a plug-in built from another revision of these headers must be rebuilt, never loaded) */
inline int gpu_abi_value() {
    return VSR_PLUGIN_ABI * 100000 + (int)((sizeof(ExpandParams) * 131 + sizeof(DevCounters) * 17 + sizeof(RecHdr) + VSR_BUCKET * 3) % 100000);
}

template <class L> struct GpuThunks {
    static cudaError_t prepare(int* blocks_per_sm) {
        cudaError_t e = cudaFuncSetAttribute(expand_kernel<L, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(typename ExpandCfg<L>::Smem));
        if (e == cudaSuccess) e = cudaFuncSetAttribute(expand_kernel<L, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(typename ExpandCfg<L>::Smem));
        if (e == cudaSuccess) e = cudaFuncSetAttribute(expand_kernel<L, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(typename ExpandCfg<L>::Smem));
        if (e != cudaSuccess) return e;
        int a = 0, b = 0;
        e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&a, expand_kernel<L, false>, ExpandCfg<L>::WARPS * 32, sizeof(typename ExpandCfg<L>::Smem));
        if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, expand_kernel<L, true>, ExpandCfg<L>::WARPS * 32, sizeof(typename ExpandCfg<L>::Smem));
        *blocks_per_sm = a < b ? a : b;
        return e;
    }
    static cudaError_t launch_expand(const ExpandParams& p, int grid, cudaStream_t st) {
        /* the one-GPU instantiation has no drain: records to insert (drain_total) need the MULTI one at any world size.
           Coverage has one instantiation per layout, the MULTI one, for every launch of a run that counts (one more kernel
           to compile per layout, not two); the grid and the block are the same for all three */
        if (p.cover) expand_kernel<L, true, true><<<grid, ExpandCfg<L>::WARPS * 32, sizeof(typename ExpandCfg<L>::Smem), st>>>(p);
        else if (p.world > 1 || p.drain_total) expand_kernel<L, true><<<grid, ExpandCfg<L>::WARPS * 32, sizeof(typename ExpandCfg<L>::Smem), st>>>(p);
        else expand_kernel<L, false><<<grid, ExpandCfg<L>::WARPS * 32, sizeof(typename ExpandCfg<L>::Smem), st>>>(p);
        return cudaGetLastError();
    }
    static cudaError_t launch_patch(const ExpandParams& p, const uint8_t* ties, unsigned long long ntie, unsigned long long n_out, cudaStream_t st) {
        if (!n_out) return cudaSuccess;
        patch_ties_kernel<L><<<(unsigned)((n_out + 255) / 256), 256, 0, st>>>(p, ties, ntie, n_out);
        return cudaGetLastError();
    }
    static cudaError_t launch_simulate(const SimParams& q, int grid, cudaStream_t st) {
        simulate_kernel<L><<<grid, 128, 0, st>>>(q);
        return cudaGetLastError();
    }
    static cudaError_t launch_audit(const ExpandParams& p, unsigned long long n_states, AuditSums* out, int sms, cudaStream_t st) {
        audit_table_kernel<<<sms * 8, 256, 0, st>>>(p.table, p.table_cap, p.level, out);
        if (n_states) audit_frontier_kernel<L><<<sms * 8, 256, 0, st>>>(p, n_states, out);
        return cudaGetLastError();
    }
    static cudaError_t launch_live_collect(const LiveParams& q, int sms, cudaStream_t st) {
        if (!q.n_in) return cudaSuccess;
        const unsigned long long want = (q.n_in + 255) / 256, most = (unsigned long long)sms * 8;
        live_collect_kernel<L><<<(unsigned)(want < most ? want : most), 256, 0, st>>>(q);
        return cudaGetLastError();
    }
    static cudaError_t launch_live_sweep(const LiveParams& q, int sms, cudaStream_t st) {
        if (!q.n) return cudaSuccess;
        const unsigned long long want = (q.n + 127) / 128, most = (unsigned long long)sms * 16;
        live_sweep_kernel<L><<<(unsigned)(want < most ? want : most), 128, 0, st>>>(q);
        return cudaGetLastError();
    }
    static uint32_t chk(const uint32_t* w, int use_view) { return check_hash<L>(w, use_view != 0); }
    static const GpuOps* get() {
        typedef ExpandCfg<L> Cfg;
        static const GpuOps ops = {chk, L::R, L::V, L::K, L::NW, L::BYTES, (int)(L::BYTES + sizeof(RecHdr)), sizeof(typename Cfg::Smem), Cfg::WARPS * 32,
                                   launch_expand, launch_patch, (int)(sizeof(TieRec) + L::BYTES), prepare, launch_simulate,
                                   Cfg::WARPS, Cfg::BLOCKS, Cfg::PASSES, Expander<L, false>::SROWS, launch_audit,
                                   launch_live_collect, launch_live_sweep};
        return &ops;
    }
};

} // namespace vsr
#endif
