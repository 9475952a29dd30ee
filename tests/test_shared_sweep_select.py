"""Which `lgssm_shared_kernel` instantiation a shared-model call launches (csrc/rxg_sweep_select.h).

The selection is plain C++; a host harness (tests/c/sweep_select_host.cpp) compiles it and the tests below hold every
pick, for every register shape and every combination of what a call observes, to a table written from the dispatch
rules.  The test sweep of tests/test_shared_sweep_variants.py cannot tell a wrong pick from a right one (the CPT, stash
and checkpoint variants are bit-identical), so this is what pins the selection.  With a built librxgauss.so it also
checks that the library instantiates exactly the picks the selection can return."""
import ctypes
import itertools
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = [(1, 1), (2, 1), (2, 2), (3, 3), (4, 1), (4, 2), (4, 4), (6, 6)]
NONE, SHARED, PER_CHAIN = 0, 1, 2          # rxg::InputSeq
FIELDS = ("cpt", "smooth", "evid", "offset", "ckpt", "peer", "useq")


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no host C++ compiler")
    so = str(tmp_path_factory.mktemp("sweep_select") / "sweep_select_host.so")
    src = os.path.join(ROOT, "tests", "c", "sweep_select_host.cpp")
    subprocess.run([cxx, "-O1", "-std=c++17", "-Wall", "-Werror", "-shared", "-fPIC", "-o", so, src], check=True)
    lib = ctypes.CDLL(so)
    lib.sweep_select.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_longlong, ctypes.c_int, ctypes.c_longlong] + \
        [ctypes.c_int] * 6 + [ctypes.c_longlong, ctypes.POINTER(ctypes.c_int)]
    lib.sweep_pick.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_int)]
    return lib


def _select(lib, *args):
    out = (ctypes.c_int * 7)()
    lib.sweep_select(*args, out)
    return tuple(out)


def _expected(d, m, batch, sm_count, force_cpt, aligned16, smooth, evid, offset, inp, peer_out, variant):
    """The dispatch rules, restated: (cpt, smooth, evid, offset, ckpt, peer, useq)."""
    cpt = 2 if batch >= sm_count * 64 * 2 else 1                 # >= ~2 resident warps per SM sub-partition
    if force_cpt > 0:
        cpt = force_cpt
    cpt = 2 if cpt >= 2 and aligned16 and batch % 2 == 0 else 1  # CPT 2 needs an even batch and 16-byte aligned buffers
    ckpt = smooth and d * d <= 16 and cpt == 2 and variant != 1  # variant 1: the stash
    if inp == PER_CHAIN:                                         # streamed beside y: no offset, no peer stores
        return (cpt, smooth, evid, 0, ckpt, 0, 1)
    if inp == SHARED and evid:                                   # table offsets + the evidence form reading u_t
        return (cpt, smooth, 1, 1, ckpt, 0, 2)
    off = offset or inp == SHARED                                # a shared sequence without evidence: the offset sweep
    peer = smooth and not evid and not off and inp == NONE and peer_out
    return (cpt, smooth, evid, off, ckpt, peer, 0)


# batch around the CPT 2 threshold (132 SMs: 16 896 chains; 114 SMs: 14 592), odd and even
BATCHES = (1, 2, 70, 71, 14591, 14592, 16895, 16896, 16897, 65536)
GRID = list(itertools.product(BATCHES, (132, 114), (0, 1, 2, 4), (0, 1), (0, 1), (0, 1), (0, 1), (NONE, SHARED, PER_CHAIN),
                              (0, 1), (0, 1, 3, 4)))


def _picks(lib, d, m):
    picks = set()
    for args in GRID:
        got = _select(lib, d, m, *args)
        want = tuple(int(v) for v in _expected(d, m, *args))
        assert got == want, f"d={d} m={m} (batch, sm_count, force_cpt, aligned16, smooth, evid, offset, input, peer_out, " \
                            f"sweep_variant)={args}: {dict(zip(FIELDS, got))} != {dict(zip(FIELDS, want))}"
        picks.add(got)
    return picks


def _instantiated(lib, d, m):
    out = (ctypes.c_int * 7)()
    inst = set()
    for i in range(lib.sweep_pick_count()):
        r = lib.sweep_pick(d, m, i, out)
        assert r in (0, 1), f"pick index {i} does not round-trip"
        if r:
            inst.add(tuple(out))
    return inst


@pytest.mark.parametrize("d,m", SHAPES)
def test_selection_matches_rules_and_instantiated_set(host, d, m):
    """Every pick equals the rules' answer, and the picks over all inputs are exactly the instantiated set."""
    picks = _picks(host, d, m)
    assert picks == _instantiated(host, d, m)
    assert len(picks) == (38 if d * d <= 16 else 30)


def _library_sweep_kernels(lib_path, cuobjdump):
    syms = subprocess.run([cuobjdump, "-symbols", lib_path], check=True, capture_output=True, text=True).stdout
    pat = re.compile(r"_ZN3rxg19lgssm_shared_kernelILi(\d+)ELi(\d+)ELi(\d+)ELi(\d+)ELb([01])ELb([01])ELb([01])ELb([01])"
                     r"ELb([01])ELi(\d+)EE")
    kernels = set()
    for mt in pat.finditer(syms):
        d, m, cpt, pf, sm, ev, of, ck, peer, useq = (int(v) for v in mt.groups())
        kernels.add((d, m, pf, (cpt, sm, ev, of, ck, peer, useq)))
    return kernels


def test_library_instantiates_exactly_the_selectable_sweeps(host):
    lib_path = os.environ.get("RXG_LIB") or os.path.join(ROOT, "rxinfer.jl_b200", "librxgauss.so")
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(lib_path) or not os.path.exists(cuobjdump):
        pytest.skip("needs a built librxgauss.so and cuobjdump")
    want = {(d, m, 4, p) for d, m in SHAPES for p in _picks(host, d, m)}
    got = _library_sweep_kernels(lib_path, cuobjdump)
    assert len(want) == 296
    extra, missing = sorted(got - want), sorted(want - got)
    assert not extra and not missing, (f"{len(extra)} instantiated but never selected (d, m, PF, pick), e.g. {extra[:4]}; "
                                       f"{len(missing)} selectable but not instantiated: {missing[:4]}")
