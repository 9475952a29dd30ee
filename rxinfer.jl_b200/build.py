"""Builds librxgauss.so (sm_90a) in-tree with nvcc.  No torch extension machinery: the product
is a plain C-ABI shared library (include/rxgauss.h) that any host (Julia ccall, ctypes, C) binds.
"""
from __future__ import annotations

import concurrent.futures as cf
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "librxgauss.so")
LGSSM_SHAPES = [(1, 1), (2, 1), (2, 2), (3, 3), (4, 1), (4, 2), (4, 4), (6, 6)]
# (source, object stem, extra flags): rxg_lgssm.cu is compiled once per (d, m) shape (explicit instantiation) + once for the dispatch
# rxg_lgssm_vmp.cu likewise once per Wishart dimension m (d = 1..6 each) + once for the C entry
UNITS = ([("rxg_lgssm.cu", f"rxg_lgssm_d{d}m{m}", (f"-DRXG_INST_D={d}", f"-DRXG_INST_M={m}")) for d, m in reversed(LGSSM_SHAPES)] +
         [("rxg_lgssm_vmp.cu", f"rxg_lgssm_vmp_m{m}", (f"-DRXG_VMP_M={m}",)) for m in range(6, 0, -1)] +
         [(s, s.replace(".cu", ""), ()) for s in
          ("rxg_lgssm_large.cu", "rxg_lgssm.cu", "rxg_umma_sweep.cu", "rxg_api.cu", "rxg_peer.cu", "rxg_rules.cu", "rxg_hgf.cu",
           "rxg_lgssm_general.cu", "rxg_lgssm_generic.cu", "rxg_lar.cu", "rxg_rules_large.cu", "rxg_predict.cu",
           "rxg_lgssm_vmp.cu", "rxg_mixture.cu", "rxg_hmm.cu", "rxg_hgf_learn.cu", "rxg_hmm_gauss.cu", "rxg_polya.cu",
           "rxg_multinomial.cu", "rxg_delta.cu")] +
         [("rxg_hostfill.cpp", "rxg_hostfill", ())])        # plain C++ (g++): host-side covariance broadcast
SOURCES = sorted({u[0] for u in UNITS})
HEADERS = ["rxg_internal.h", "rxg_linalg.cuh", "rxg_gain.cuh", "rxg_lgssm_common.cuh", "rxg_chain_step.cuh", "rxg_lgssm_shared.cuh", "rxg_lgssm_seg.cuh", "rxg_lgssm_cluster.cuh", "rxg_sweep_select.h", "rxg_umma.cuh", "rxg_lar.cuh", "rxg_hmm.cuh", "rxg_hgf_learn.cuh", "rxg_hmm_gauss.cuh", "rxg_normal_wishart.cuh", "rxg_polya.cuh", "rxg_multinomial.cuh", "rxg_delta.cuh", os.path.join("..", "..", "include", "rxgauss.h")]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-mavx2", "-Xcompiler", "-pthread", "--expt-relaxed-constexpr", "-Xptxas", "-v",
]


def _nvcc():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: librxgauss cannot be built (there is no CPU fallback)")


def embed_delta_header(objdir: str) -> str:
    """rxg_delta.cuh as the byte array ``rxg_delta_header_src`` (NUL-terminated) in an object of its own: the library
    compiles it, with the user's functions, at run time (rxg_delta.cu)."""
    with open(os.path.join(CSRC, "rxg_delta.cuh"), "rb") as f:
        data = f.read() + b"\0"
    src = os.path.join(objdir, "rxg_delta_header.cpp")
    rows = ",\n".join(",".join(str(b - 256 if b > 127 else b) for b in data[i:i + 32]) for i in range(0, len(data), 32))
    with open(src, "w") as f:
        f.write(f"extern const char rxg_delta_header_src[] = {{\n{rows}\n}};\n")
    obj = os.path.join(objdir, "rxg_delta_header.o")
    r = subprocess.run(["g++", "-O0", "-fPIC", "-c", src, "-o", obj], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"compiling the embedded Delta header failed:\n{r.stderr}")
    return obj


def _stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False, extra_flags=(), lib: str = LIB, objdir_name: str = "build") -> str:
    """``extra_flags`` / ``lib`` / ``objdir_name`` build an A/B variant next to the product library (tuning
    experiments, e.g. ``extra_flags=("-DSOME_SWITCH=1",), lib=".../librxgauss_b.so"``, selected at run time with RXG_LIB=<path>)."""
    if not force and lib == LIB and not _stale():
        return LIB
    nvcc = _nvcc()
    objdir = os.path.join(HERE, objdir_name)
    os.makedirs(objdir, exist_ok=True)

    def compile_one(unit):
        src, stem, defs = unit
        obj = os.path.join(objdir, stem + ".o")
        if src.endswith(".cpp"):
            cmd = ["g++", "-O3", "-std=c++17", "-fPIC", "-pthread", "-Wall", "-c", os.path.join(CSRC, src), "-o", obj]
        else:
            cmd = [nvcc, *NVCC_FLAGS, *extra_flags, *defs, "-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        log = os.path.join(objdir, stem + ".ptxas.log")
        with open(log, "w") as f:
            f.write(r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            print(r.stderr)
        return obj

    with cf.ThreadPoolExecutor(max_workers=min(len(UNITS), os.cpu_count() or 4)) as ex:
        objs = list(ex.map(compile_one, UNITS))
    objs.append(embed_delta_header(objdir))
    tmp = lib + ".tmp"      # link next to the target and rename: a concurrent reader never sees a partial file
    cmd = [nvcc, "-shared", "-o", tmp, *objs, "-ldl", "-lpthread", "-Xcompiler", "-fPIC"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    os.replace(tmp, lib)
    return lib


if __name__ == "__main__":
    import sys
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
