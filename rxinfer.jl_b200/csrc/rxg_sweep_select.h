// Which lgssm_shared_kernel instantiation a shared-model call launches (rxg_lgssm.cu: launch_shared).
//
// Plain C++ with no CUDA types, so that the dispatcher and a host-compiled test (tests/test_shared_sweep_select.py) use
// the same function.  select_shared_sweep maps what the call observes to the template values of the kernel;
// sweep_pick_reachable describes the set it can return for a (d, m) shape, and only that set is instantiated.
#pragma once
#include <stdint.h>

namespace rxg {

enum class InputSeq : int { none = 0, shared = 1, per_chain = 2 };   // RXG_U_SEQ_SHARED / RXG_U_SEQ_CHAIN

struct SweepQuery {
    int d, m;
    int64_t batch;
    int sm_count;
    long long force_cpt;     // RXG_OPT_FORCE_CPT (0: automatic)
    bool aligned16;          // every per-chain buffer the sweep streams is 16-byte aligned
    bool smooth, evid;
    bool offset;             // a nonzero constant transition offset u
    InputSeq input;
    bool peer_out;           // fused all-gather destinations are present (c.po)
    long long sweep_variant; // RXG_OPT_SWEEP_VARIANT (1: the stash instead of checkpoint + recompute)
};

// The template values <CPT, SMOOTH, EVID, OFFSET, CKPT, PEER, USEQ> of lgssm_shared_kernel (PF is fixed at 4).
struct SweepPick {
    int cpt;
    bool smooth, evid, offset, ckpt, peer;
    int useq;                // 0: none, 1: per-chain sequence, 2: shared sequence with evidence
};

constexpr SweepPick select_shared_sweep(const SweepQuery& q) {
    // chains per thread: keep >= ~2 resident warps per SM sub-partition; wider per-thread vectors cut the number of
    // (128-byte-per-warp) store instructions per byte.  CPT = 2 needs an even batch and 16-byte aligned buffers.
    int cpt = (q.batch >= (int64_t)q.sm_count * 64 * 2) ? 2 : 1;
    if (q.force_cpt > 0) cpt = (int)q.force_cpt;            // test / tuning override
    SweepPick p{};
    p.cpt = (cpt >= 2 && q.aligned16 && q.batch % 2 == 0) ? 2 : 1;
    p.smooth = q.smooth;
    p.evid = q.evid;
    // checkpoint + recompute instead of the forward->backward stash; with one chain per thread the stash is faster
    // and larger states exceed the kernel's static shared memory
    p.ckpt = q.smooth && q.d * q.d <= 16 && p.cpt == 2 && q.sweep_variant != 1;
    if (q.input == InputSeq::per_chain) {
        p.useq = 1;          // streamed beside y; the gain tables carry no offsets
    } else if (q.input == InputSeq::shared && q.evid) {
        p.useq = 2;          // the tables carry the offsets, the explicit evidence form reads u_t
        p.offset = true;
    } else {
        p.offset = q.offset || q.input == InputSeq::shared;   // a shared sequence lives in the tables' offset terms
        // fused all-gather: only the headline variant (smoothing, no evidence, no offset) has a PEER instantiation
        p.peer = q.smooth && !q.evid && !p.offset && q.input == InputSeq::none && q.peer_out;
    }
    return p;
}

constexpr bool sweep_pick_reachable(int d, int m, const SweepPick& p) {
    (void)m;
    if (p.cpt != 1 && p.cpt != 2) return false;
    if (p.ckpt && !(p.smooth && d * d <= 16 && p.cpt == 2)) return false;
    if (p.peer && !(p.smooth && !p.evid && !p.offset && p.useq == 0)) return false;
    if (p.useq == 1) return !p.offset;
    if (p.useq == 2) return p.evid && p.offset;
    return p.useq == 0;
}

// A dense index over every SweepPick (unreachable ones included), for dispatch over a std::make_integer_sequence.
constexpr int SWEEP_PICK_COUNT = 3 << 6;
constexpr int sweep_pick_index(const SweepPick& p) {
    return (p.cpt == 2 ? 1 : 0) | p.smooth << 1 | p.evid << 2 | p.offset << 3 | p.ckpt << 4 | p.peer << 5 | p.useq << 6;
}
constexpr SweepPick sweep_pick_at(int i) {
    return SweepPick{(i & 1) ? 2 : 1, (i & 2) != 0, (i & 4) != 0, (i & 8) != 0, (i & 16) != 0, (i & 32) != 0, i >> 6};
}

}  // namespace rxg
