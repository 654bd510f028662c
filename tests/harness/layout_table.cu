/*
 * layout_table.cu — what every Layout<R, V, K> in the packed encoding's range would be, and whether it can be built.
 *
 * Host only: it instantiates the layouts' sizes and constexprs (vsr_layout.h, ExpandCfg of vsr_gpu.cuh), never a kernel, so
 * it compiles in seconds for all 630 layouts.  The limits are ExpandCfg's own constants, which the expand kernel and
 * vsr_layout_plugin.cu assert.  One line per layout, whitespace separated, after a header line naming the columns:
 *   R V L            ReplicaCount, |Values|, StartViewOnTimerLimit (K = L + 1)
 *   nw ncand maxgrp  32-bit words of a packed state, (action, binding) candidates, the largest action group
 *   msgs             message slots: the most messages a state can hold in the flat form (VSR_MAX_MSGS)
 *   warps blocks passes smem rows   the expand kernel's shape: ExpandCfg's WARPS, BLOCKS, PASSES, sizeof(Smem), staging rows
 *   state_ok smem_ok pool_ok        the plug-in's limits: state bytes <= VSR_MAX_STATE_BYTES, Smem fits one SM, the
 *                                   pool item and the scan's packed counters fit 16 bits
 * build: nvcc -gencode arch=compute_90a,code=sm_90a -std=c++17 -I../../vsr-tlaplus_b200/csrc layout_table.cu
 */
#include <cstdio>
#include <utility>

#include "../../include/vsr_b200.h"
#include "vsr_gpu.cuh"

template <int I> static void row() {
    constexpr int R = 2 + I / (7 * 15), V = 1 + I / 15 % 7, K = 1 + I % 15;
    typedef vsr::Layout<R, V, K> L;
    typedef vsr::ExpandCfg<L> Cfg;
    typedef typename Cfg::Smem Smem;
    constexpr int rows = (int)(sizeof(std::declval<typename Smem::Stage&>().tstage) / sizeof(unsigned long long));
    constexpr int msgs = L::NSVC + L::NDVC + L::NSV + V * L::O + L::NPOK + 2 * L::NGS;
    printf("%d %d %d %d %d %d %d %d %d %d %zu %d %d %d %d\n", R, V, K - 1, L::NW, L::NCAND, Cfg::max_grp(), msgs, Cfg::WARPS,
           Cfg::BLOCKS, Cfg::PASSES, sizeof(Smem), rows, L::BYTES <= VSR_MAX_STATE_BYTES, sizeof(Smem) <= Cfg::SMEM_SM,
           Cfg::POOL_ITEM_FITS && Cfg::POOL_COUNTERS_FIT);
}
template <int... I> static void rows(std::integer_sequence<int, I...>) { (row<I>(), ...); }

int main() {
    printf("R V L nw ncand maxgrp msgs warps blocks passes smem rows state_ok smem_ok pool_ok\n");
    rows(std::make_integer_sequence<int, 6 * 7 * 15>());
    return 0;
}
