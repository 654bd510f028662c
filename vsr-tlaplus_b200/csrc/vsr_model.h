/*
 * vsr_model.h — internal: the run-time face of one compile-time Layout<R,V,K>, and the model object
 * behind the opaque VsrModel of include/vsr_b200.h.
 */
#ifndef VSR_MODEL_H
#define VSR_MODEL_H

#include <string>
#include <vector>

#include "../../include/vsr_b200.h"
#include "vsr_actions.h"

/* (ReplicaCount, |Values|, 1 + StartViewOnTimerLimit) combinations compiled in.  BASELINE.json
   configs: (2,1,2) cfg1, (3,2,3) cfg2 = shipped VSR.cfg, (3,3,4) cfg3 = README, (5,2,3) cfg4. */
#ifdef VSR_ONLY_R /* kernel experiments: -DVSR_ONLY_R=3 -DVSR_ONLY_V=2 -DVSR_ONLY_K=3 compiles one layout in seconds */
#define VSR_FOR_EACH_CONFIG(X) X(VSR_ONLY_R, VSR_ONLY_V, VSR_ONLY_K)
#else
#define VSR_FOR_EACH_CONFIG(X) \
    X(2, 1, 2) X(2, 2, 2) X(2, 2, 3) X(2, 3, 3) X(3, 1, 2) X(3, 1, 3) X(3, 2, 2) X(3, 2, 3) X(3, 2, 4) X(3, 3, 2) X(3, 3, 3) \
    X(3, 3, 4) X(4, 1, 2) X(4, 2, 2) X(4, 2, 3) X(4, 3, 3) X(5, 1, 2) X(5, 2, 2) X(5, 2, 3) X(5, 3, 3)
#endif

namespace vsr {

struct GpuOps; /* vsr_gpu.cu */

/* vsr_model_create's `invariant` bits above the INVARIANT mask (include/vsr_b200.h).  MODEL_MAJORITY_FIRST_BIT is the whole
   INVARIANT order this entry point can express: NoLogDivergence (4) and TestInv (8) never fail (VSR.tla:926-931, :952), so
   only the order of bits 1 and 2 can change the name reported; a third invariant that can fail needs a full order here */
enum { MODEL_PROPERTY_BIT = 512, MODEL_HOOK_Q_BIT = 1024, MODEL_HOOK_INIT_EDGE_BIT = 2048, MODEL_MAJORITY_FIRST_BIT = 4096 };
/* names of the INVARIANT mask bits 1, 2, 4, 8 */
static const char* const INVARIANT_NAMES[4] = {"AcknowledgedWriteNotLost", "AcknowledgedWritesExistOnMajority", "NoLogDivergence", "TestInv"};
enum { LIVE_HOOK_Q = 1, LIVE_HOOK_INIT_EDGE = 2 };

struct ModelOps {
    int R, V, K, nw, bytes, bits, ncand;
    void (*init)(uint32_t*);
    int (*step)(const RunCfg*, const uint32_t*, int, uint32_t*);
    int (*guard)(const RunCfg*, const uint32_t*, int);
    int (*action_of)(int);
    int (*invariant)(const RunCfg*, const uint32_t*);
    uint64_t (*fingerprint)(const uint32_t*, int use_view);
    uint32_t (*aux_key)(const uint32_t*);
    int (*canon)(uint32_t*);
    int (*unpack)(const uint32_t*, VsrFlatState*);
    int (*pack)(const VsrFlatState*, uint32_t*, int symmetry);
    int (*literal_cand)(const uint32_t*, int cand);
    uint64_t (*fingerprint_bytewise)(const uint32_t*, int use_view);
    int (*random_enabled)(const RunCfg*, const uint32_t*, uint64_t* rng);
    int (*enabled_list)(const RunCfg*, const uint32_t*, uint32_t* out); /* register-mask form of the guards (the kernel's scan) */
    int (*property)(const RunCfg*, const uint32_t*, int live_hooks);   /* the liveness pass's state predicate (live_pred) */
};
/* bump when ModelOps / GpuOps / ExpandParams / LiveParams / ReshardParams / SimParams change shape: a layout plug-in built against another value is rebuilt */
#define VSR_PLUGIN_ABI 14
const ModelOps* find_model_ops(int R, int V, int K);
const GpuOps* find_gpu_ops(int R, int V, int K); /* defined in vsr_gpu.cu */

} // namespace vsr

extern "C" int vsr_gpu_abi(void); /* vsr_gpu.cu: version + shapes of the kernel parameter structs */

struct VsrModel {
    VsrModelInfo info;
    vsr::RunCfg run;
    const vsr::ModelOps* ops;
    const vsr::GpuOps* gpu;
    int check_deadlock_cfg; /* CHECK_DEADLOCK in the cfg: -1 unset */
    int live_hooks = 0;     /* test hooks of the liveness pass (vsr_model_create): LIVE_HOOK_* */
    std::vector<int> inv_order; /* INVARIANT mask bits in the config's order: TLC reports the first one a state violates */
    std::string action_location[VSR_NUM_ACTIONS];
};

#endif
