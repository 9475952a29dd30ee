// Test harness (NOT part of librxgauss.so): the shared-sweep selection (csrc/rxg_sweep_select.h) compiled for the host,
// so that tests/test_shared_sweep_select.py can check every pick the dispatcher makes without a GPU.
#include "../../rxinfer.jl_b200/csrc/rxg_sweep_select.h"

static void put(const rxg::SweepPick& p, int* out) {
    out[0] = p.cpt; out[1] = p.smooth; out[2] = p.evid; out[3] = p.offset; out[4] = p.ckpt; out[5] = p.peer; out[6] = p.useq;
}

// out[7] = <CPT, SMOOTH, EVID, OFFSET, CKPT, PEER, USEQ>
extern "C" void sweep_select(int d, int m, long long batch, int sm_count, long long force_cpt, int aligned16, int smooth,
                             int evid, int offset, int input, int peer_out, long long sweep_variant, int* out) {
    rxg::SweepQuery q = {};
    q.d = d; q.m = m; q.batch = batch; q.sm_count = sm_count; q.force_cpt = force_cpt; q.aligned16 = aligned16 != 0;
    q.smooth = smooth != 0; q.evid = evid != 0; q.offset = offset != 0; q.input = (rxg::InputSeq)input;
    q.peer_out = peer_out != 0; q.sweep_variant = sweep_variant;
    put(rxg::select_shared_sweep(q), out);
}

// Pick index `index` of the dispatcher's enumeration: writes the pick and returns 1 if it is instantiated for (d, m),
// 0 if not, and -1 if the index does not round-trip.
extern "C" int sweep_pick(int d, int m, int index, int* out) {
    const rxg::SweepPick p = rxg::sweep_pick_at(index);
    put(p, out);
    if (rxg::sweep_pick_index(p) != index) return -1;
    return rxg::sweep_pick_reachable(d, m, p) ? 1 : 0;
}

extern "C" int sweep_pick_count() { return rxg::SWEEP_PICK_COUNT; }
