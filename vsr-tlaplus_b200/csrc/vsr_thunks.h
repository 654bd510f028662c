/*
 * vsr_thunks.h — internal: the run-time vtable (ModelOps, vsr_model.h) of one compile-time Layout<R,V,K>.
 * Instantiated for every built-in layout in vsr_host.cpp and for one layout in a layout plug-in
 * (vsr_layout_plugin.cu).
 */
#ifndef VSR_THUNKS_H
#define VSR_THUNKS_H

#include "vsr_flat_conv.h"
#include "vsr_model.h"

namespace vsr {

inline const uint64_t* fp64_table() {
    static uint64_t tab[8 * 256]; /* slicing-by-8 tables; the first 256 entries are the byte table */
    static bool built = false;
    if (!built) { fp64_build_slices(tab); built = true; }
    return tab;
}

template <class L> struct Thunks {
    static void init(uint32_t* w) { Ops<L>::init(w); }
    static int step(const RunCfg* run, const uint32_t* s, int cand, uint32_t* n) { return Ops<L>::template step<true>(*run, s, cand, n); }
    static int guard(const RunCfg* run, const uint32_t* s, int cand) { return Ops<L>::template step<false>(*run, s, cand, nullptr); }
    static int action_of(int cand) { return Ops<L>::action_of(cand); }
    static int invariant(const RunCfg* run, const uint32_t* w) { return Ops<L>::invariant(*run, w); }
    static uint64_t fingerprint(const uint32_t* w, int use_view) { return fp64_view8<L>(fp64_table(), w, use_view != 0); }
    static int random_enabled(const RunCfg* run, const uint32_t* s, uint64_t* rng) { return Ops<L>::random_enabled(*run, s, *rng); }
    static int enabled_list(const RunCfg* run, const uint32_t* s, uint32_t* out) { return Ops<L>::enabled_list(*run, s, out); }
    static uint64_t fingerprint_bytewise(const uint32_t* w, int use_view) { return fp64_view<L>(fp64_table(), w, use_view != 0); }
    static uint32_t aux_key(const uint32_t* w) { return Ops<L>::aux_key(w); }
    static int canon(uint32_t* w) { return Ops<L>::canonicalize(w); }
    static int unpack(const uint32_t* w, VsrFlatState* f) { return Conv<L>::unpack(w, f); }
    static int pack(const VsrFlatState* f, uint32_t* w, int sym) { return Conv<L>::pack(f, w, sym != 0); }
    static int literal_cand(const uint32_t* w, int cand) { return Ops<L>::literal_cand(w, cand); }
    static int property(const RunCfg* run, const uint32_t* w, int live_hooks) { return Ops<L>::live_pred(*run, w, live_hooks) ? 1 : 0; }
    static const ModelOps* get() {
        static const ModelOps ops = {L::R, L::V, L::K, L::NW, L::BYTES, L::TOTAL_BITS, L::NCAND, init, step, guard,
                                     action_of, invariant, fingerprint, aux_key, canon, unpack, pack, literal_cand, fingerprint_bytewise, random_enabled, enabled_list,
                                     property};
        return &ops;
    }
};

} // namespace vsr
#endif
