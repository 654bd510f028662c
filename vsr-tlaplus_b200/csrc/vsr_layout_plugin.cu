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
static_assert(PluginLayout::BYTES <= VSR_MAX_STATE_BYTES, "packed state larger than the C ABI's VSR_MAX_STATE_BYTES");
static_assert(VSR_ONLY_R <= VSR_MAX_R && VSR_ONLY_V <= VSR_MAX_V, "beyond the flat interchange form (include/vsr_flat.h)");
static_assert(sizeof(vsr::ExpandCfg<PluginLayout>::Smem) <= 227 * 1024, "expand kernel's shared memory exceeds an SM");

extern "C" {
int vsr_plugin_abi(void) { return vsr::gpu_abi_value(); }
const vsr::ModelOps* vsr_plugin_model_ops(void) { return vsr::Thunks<PluginLayout>::get(); }
const vsr::GpuOps* vsr_plugin_gpu_ops(void) { return vsr::GpuThunks<PluginLayout>::get(); }
}
