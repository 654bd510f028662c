/*
 * vsr_layout_plugin.cu — one Layout<R,V,K> as a loadable module.
 *
 * libvsr_b200.so carries the layouts of VSR_FOR_EACH_CONFIG (vsr_model.h).  The reference tells its user to edit the
 * constants of VSR.cfg (README.md:11-18 of the reference); for constants outside that list the loader (vsr_host.cpp,
 * load_layout_plugin) compiles this file once with
 *     nvcc -gencode arch=compute_90a,code=sm_90a -DVSR_ONLY_R=<ReplicaCount> -DVSR_ONLY_V=<|Values|>
 *          -DVSR_ONLY_K=<1 + StartViewOnTimerLimit> -shared -o layouts/libvsr_layout_R_V_K.so vsr_layout_plugin.cu
 * and takes the two vtables from it.  Same templates as the built-in layouts: nothing here but the instantiation.
 */
#include "vsr_gpu_thunks.cuh"
#include "vsr_thunks.h"

#if !defined(VSR_ONLY_R) || !defined(VSR_ONLY_V) || !defined(VSR_ONLY_K)
#error "compile with -DVSR_ONLY_R=.. -DVSR_ONLY_V=.. -DVSR_ONLY_K=.."
#endif

typedef vsr::Layout<VSR_ONLY_R, VSR_ONLY_V, VSR_ONLY_K> PluginLayout;
typedef vsr::ExpandCfg<PluginLayout> PluginCfg;
static_assert(VSR_ONLY_R <= VSR_MAX_R && VSR_ONLY_V <= VSR_MAX_V, "beyond the flat interchange form (include/vsr_flat.h)");

/* The layout's compile-time limits, each checked in a class whose name carries the numbers: the compiler prints that name
   with a failed assertion ("detected during instantiation of class "vsr_limit_state_bytes<BYTES, MAX> [with BYTES=288,
   MAX=256]""), and the loader turns that into a one-line message (vsr_host.cpp, plugin_limit_message). */
template <int BYTES, int MAX> struct vsr_limit_state_bytes {
    static_assert(BYTES <= MAX, "packed state larger than the C ABI's VSR_MAX_STATE_BYTES");
};
template <size_t BYTES, size_t MAX> struct vsr_limit_smem_bytes {
    static_assert(BYTES <= MAX, "expand kernel's shared memory exceeds an SM");
};
template <int GROUP, int MAX, bool FITS> struct vsr_limit_pool_item {
    static_assert(FITS, "an action group does not fit the expand kernel's 16-bit pool items");
};
/* the largest action group the pool item (candidate offset: 16 - TBITS bits) and the scan's packed counters hold */
constexpr int kPluginMaxGroup = (1 << (16 - PluginCfg::TBITS)) - 1 < 65535 / PluginCfg::NS ? (1 << (16 - PluginCfg::TBITS)) - 1 : 65535 / PluginCfg::NS;
template struct vsr_limit_state_bytes<PluginLayout::BYTES, VSR_MAX_STATE_BYTES>;
template struct vsr_limit_smem_bytes<sizeof(PluginCfg::Smem), PluginCfg::SMEM_SM>;
template struct vsr_limit_pool_item<PluginCfg::max_grp(), kPluginMaxGroup, PluginCfg::POOL_ITEM_FITS && PluginCfg::POOL_COUNTERS_FIT>;

extern "C" {
int vsr_plugin_abi(void) { return vsr::gpu_abi_value(); }
const vsr::ModelOps* vsr_plugin_model_ops(void) { return vsr::Thunks<PluginLayout>::get(); }
const vsr::GpuOps* vsr_plugin_gpu_ops(void) { return vsr::GpuThunks<PluginLayout>::get(); }
}
