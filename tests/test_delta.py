"""Delta node on the CPU: the fp64 oracle reduces to the LGSSM oracle for linear maps under both methods, the library's
NVRTC path compiles the exact program it would load (embedded header, user source, generated tail) for sm_90a and
returns the compiler log for a broken source, and infer() refuses what the batched path does not run."""
import ctypes
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import delta as D
from oracle import lgssm

from delta_models import D8_SRC, PENDULUM_SRC, TRACKER_SRC
from util import TOL_COV, TOL_MEAN, rel_l2

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _linear_model(seed=0, d=3, m=2):
    rng = np.random.default_rng(seed)
    Aq, _ = np.linalg.qr(rng.standard_normal((d, d)))
    return dict(A=0.95 * Aq, B=rng.standard_normal((m, d)), P=0.1 * np.eye(d), Q=0.5 * np.eye(m),
                m0=rng.standard_normal(d), S0=2.0 * np.eye(d))


@pytest.mark.parametrize("method,ut", [("linearization", D.UT_DEFAULTS), ("unscented", D.UT_DEFAULTS),
                                       ("unscented", (0.5, 2.0, 1.0)), ("unscented", (1.0, 0.0, 3.0))])
@pytest.mark.parametrize("observe", ["B", "g"])
def test_linear_maps_reduce_to_the_lgssm_oracle(method, ut, observe):
    mod = _linear_model()
    _, y = lgssm.generate_data(mod, 40, 3, seed=5)
    mask = np.ones((40, 3), np.uint8)
    mask[7, 1] = mask[20, :] = 0
    ref = lgssm.smooth_reference_schedule(y, **mod, mask=mask)
    g = D.linear(mod["B"]) if observe == "g" else None
    r = D.smooth(y, D.linear(mod["A"]), mod["P"], mod["m0"], mod["S0"], method, g=g, B=mod["B"], Q=mod["Q"], mask=mask,
                 ut=ut)
    np.testing.assert_allclose(r["mean"], ref["mean"], rtol=0, atol=1e-9)
    np.testing.assert_allclose(r["cov"], ref["cov"], rtol=0, atol=1e-9)


def test_unscented_matches_linearization_to_second_order():
    """For a nearly linear map the two methods agree up to the curvature term (a check that the sigma-point weights
    carry the right signs)."""
    mu, S = np.array([0.3, -0.2]), 1e-4 * np.eye(2)
    a = D.moments(D.PENDULUM, mu, S, "linearization")
    b = D.moments(D.PENDULUM, mu, S, "unscented")
    for x, z in zip(a, b):
        np.testing.assert_allclose(x, z, rtol=1e-3, atol=1e-9)


def test_paper_dataset_keeps_its_quirks():
    ts, states, obs = D.dataset(50, precision=1.0, seed=42)
    assert obs[0] == 0.0 and np.all(obs[1:] != 0.0)
    np.testing.assert_allclose(states[:, 0], [0.5, 0.0])
    np.testing.assert_allclose(states[:, 1], D.PENDULUM.h(states[:, 0]))
    np.testing.assert_allclose(ts[:3], [0.01, 0.02, 0.03])
    _, _, again = D.dataset(50, precision=1.0, seed=42)
    np.testing.assert_array_equal(obs, again)


def _check(rx, src, f, g, d, m, method, ut=None):
    lib = rx._lib.load()
    log = ctypes.create_string_buffer(1 << 16)
    uta = (ctypes.c_double * 3)(*ut) if ut is not None else None
    rc = lib.rxg_delta_check_source(src.encode(), f.encode(), g.encode() if g else None, d, m, method, uta, log, len(log))
    return rc, log.value.decode()


@pytest.mark.parametrize("src,f,g,d,m,method", [
    (PENDULUM_SRC, "pendulum", None, 2, 1, 0), (PENDULUM_SRC, "pendulum", None, 2, 1, 1),
    (TRACKER_SRC, "cv", "range_bearing", 4, 2, 0), (TRACKER_SRC, "cv", "range_bearing", 4, 2, 1),
    (D8_SRC, "f8", "g8", 8, 3, 0)])
def test_nvrtc_compiles_the_program_for_sm90a(rx, src, f, g, d, m, method):
    rc, log = _check(rx, src, f, g, d, m, method)
    assert rc == rx._lib.RXG_OK, log
    assert "rxg_delta_smooth" in log and "rxg_delta_filter" in log and "sm_90a" in log   # the ptxas report


def test_every_dual_overload_compiles(rx):
    src = """
template <class S> __device__ void all(const S* x, S* z) {
    z[0] = sin(x[0]) + cos(x[1]) + tan(x[0]) * exp(x[1]) - log(x[2]) / sqrt(x[2]);
    z[1] = tanh(x[0]) + atan(x[1]) + atan2(x[0], x[1]) + atan2(x[0], 2.0) + atan2(1.0, x[1]);
    z[2] = pow(x[2], 1.5) + pow(x[2], x[0]) + pow(2.0, x[1]) + fabs(-x[0]) + 2 * x[1] - x[0] / 3.0 + 1.0f;
    if (x[0] > x[1]) z[2] += 1.0 / x[2];
}
"""
    for method in (0, 1):
        rc, log = _check(rx, src, "all", None, 3, 1, method)
        assert rc == rx._lib.RXG_OK, log


def test_syntax_error_comes_back_as_the_nvrtc_log(rx):
    rc, log = _check(rx, "template <class S> __device__ void f(const S* x, S* z) { z[0] = x[0] +; }", "f", None, 1, 1, 0)
    assert rc == rx._lib.RXG_ERR_BAD_ARG
    assert "user_source(1): error" in log


@pytest.mark.parametrize("args", [(2, 1, 7, None), (0, 1, 0, None), (9, 1, 0, None), (2, 9, 0, None),
                                  (2, 1, 1, (0.0, 2.0, 0.0))])
def test_bad_shapes_and_methods_are_refused_before_compiling(rx, args):
    d, m, method, ut = args
    rc, log = _check(rx, PENDULUM_SRC, "pendulum", None, d, m, method, ut)
    assert rc == rx._lib.RXG_ERR_BAD_ARG and log.startswith("delta:")


def test_infer_refusals(rx):
    from rxinfer_jl_b200 import inference as I
    f = I.CudaFunction(PENDULUM_SRC, "pendulum", 2, 2)
    sm = I.nonlinear_gaussian_ssm_smoothing(f=f, P=np.eye(2), Q=np.eye(1), x0=(np.zeros(2), np.eye(2)), B=[[1.0, 0.0]])
    data = {"y": np.zeros((5, 1, 2), np.float32)}
    with pytest.raises(ValueError, match="approximation method"):
        I.infer(model=sm, data=data, meta={"f": None})
    with pytest.raises(ValueError, match="need an approximation method"):
        I.infer(model=sm, data=data)
    with pytest.raises(ValueError, match="not Delta nodes"):
        I.infer(model=sm, data=data, meta={"f": I.Linearization(), "g": I.Linearization()})
    with pytest.raises(NotImplementedError, match="energy term"):
        I.infer(model=sm, data=data, meta={"f": I.Unscented()}, free_energy=True)
    with pytest.raises(NotImplementedError, match="outside the batched hot path"):
        I.infer(model=sm, datastream=[], batch=2, keephistory=3, meta={"f": I.Linearization()})
    with pytest.raises(NotImplementedError, match="per-message machinery"):       # meta stays refused elsewhere
        I.infer(model=I.hgf(), data={"y": np.zeros((3, 2))}, meta={"f": I.Linearization()})
    pend = I.nonlinear_gamma_streaming(f=f, c=[1.0, 0.0])
    with pytest.raises(NotImplementedError, match="q\\(state\\) q\\(noise\\)"):
        I.infer(model=pend, datastream=[], batch=1, meta={"f": I.Linearization()})
    tr = I.nonlinear_gaussian_ssm_smoothing(f=I.CudaFunction(TRACKER_SRC, "cv", 4, 4), P=np.eye(4), Q=np.eye(2),
                                            x0=(np.zeros(4), np.eye(4)),
                                            g=I.CudaFunction(TRACKER_SRC, "range_bearing", 4, 2))
    with pytest.raises(NotImplementedError, match="different approximation methods"):
        I.infer(model=tr, data={"y": np.zeros((3, 2, 1))}, meta={"f": I.Linearization(), "g": I.Unscented()})
    with pytest.raises(NotImplementedError, match="state0 = \\(mean, cov\\) and noise0"):   # the paper's initmarginals
        I.infer(model=pend, datastream=[], batch=1, meta={"f": I.Linearization()}, constraints=I.MeanField(),
                initialization={"state": None, "noise": None})
    with pytest.raises(NotImplementedError, match="x0 = \\(mean, cov\\)"):
        I.infer(model=sm, data=data, meta={"f": I.Linearization()}, initialization={"x": None})
    with pytest.raises(NotImplementedError, match="returnvars"):
        I.infer(model=sm, data=data, meta={"f": I.Linearization()}, returnvars={"x": I.KeepEach()})


@pytest.mark.parametrize("shape", [(5,), (3, 5), (5, 3, 1), (4, 3), (5, 4)])
def test_a_wrongly_shaped_mask_is_refused_on_the_host(rx, shape):
    """The Delta kernels read ymask[t][b] for every step and chain: anything but [T, batch] is refused before it is
    copied to the device or launched (T = 5 steps, batch = 3 chains here)."""
    from rxinfer_jl_b200.context import delta_mask
    with pytest.raises(ValueError, match=r"mask must be \[T, batch\] = \(5, 3\)"):
        delta_mask(np.ones(shape, np.uint8), 5, 3, "cpu", "delta_filter_chunk")
    ok = delta_mask(np.ones((5, 3), bool), 5, 3, "cpu", "delta_filter_chunk")
    assert ok.dtype.is_floating_point is False and tuple(ok.shape) == (5, 3)


# ------------------------------------------------------------------ the header compiled for the host (tests/c/delta_host_harness.cu)
@pytest.fixture(scope="module")
def host():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = tempfile.mkdtemp(prefix="rxg_delta_host_")
    so = os.path.join(out, "delta_host.so")
    subprocess.run([nvcc, "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "-shared", "-Xcompiler", "-fPIC", "-o", so,
                    os.path.join(ROOT, "tests", "c", "delta_host_harness.cu")], check=True)
    yield ctypes.CDLL(so)
    shutil.rmtree(out, ignore_errors=True)


def _p(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))


def _dual_reference(a, b):
    s2 = a * a + b * b
    return [
        (np.sin(a), [np.cos(a), 0]), (np.cos(a), [-np.sin(a), 0]), (np.tan(a), [1 / np.cos(a) ** 2, 0]),
        (np.exp(a), [np.exp(a), 0]), (np.log(a), [1 / a, 0]), (np.sqrt(a), [0.5 / np.sqrt(a), 0]),
        (np.tanh(a), [1 - np.tanh(a) ** 2, 0]), (np.arctan(a), [1 / (1 + a * a), 0]), (abs(b), [0, np.sign(b)]),
        (np.arctan2(a, b), [b / s2, -a / s2]), (np.arctan2(a, 2.0), [2 / (a * a + 4), 0]),
        (np.arctan2(1.5, b), [0, -1.5 / (2.25 + b * b)]), (a ** 2.5, [2.5 * a ** 1.5, 0]),
        (a ** b, [b * a ** (b - 1), a ** b * np.log(a)]), (1.7 ** b, [0, 1.7 ** b * np.log(1.7)]),
        (-a * b + a / b - 2 / b + 3 * a - 0.5, [-b + 1 / b + 3, -a - a / b ** 2 + 2 / b ** 2])]


@pytest.mark.parametrize("x", [(0.7, -1.3), (1.9, 0.4)])
def test_dual_jacobians_match_the_analytic_ones(host, x):
    xa = np.array(x, np.float32)
    val, jac = np.zeros(16, np.float32), np.zeros((16, 2), np.float32)
    assert host.delta_host_dual_ops(_p(xa), _p(val), _p(jac)) == 16
    for k, (v, j) in enumerate(_dual_reference(float(xa[0]), float(xa[1]))):
        np.testing.assert_allclose(val[k], v, rtol=2e-6, atol=1e-6, err_msg=f"value of op {k}")
        np.testing.assert_allclose(jac[k], j, rtol=2e-5, atol=1e-6, err_msg=f"Jacobian of op {k}")


def _wave(d):
    h = lambda x: 0.9 * x + 0.2 * np.sin(np.roll(x, -1))

    def jac(x):
        J = 0.9 * np.eye(d)
        for i in range(d):
            J[i, (i + 1) % d] += 0.2 * np.cos(x[(i + 1) % d])
        return J
    return D.Fn(h, jac)


def _wave_case(d, T, seed):
    rng = np.random.default_rng(seed)
    f32 = lambda a: np.asarray(a, np.float32)
    P, S0 = f32(0.05 * np.eye(d)), f32(0.5 * np.eye(d))
    m0, B, Q = f32(rng.standard_normal(d)), f32(rng.standard_normal((1, d))), f32([[0.2]])
    y = f32(np.cumsum(rng.standard_normal(T)) * 0.1)
    return P, S0, m0, B, Q, y


@pytest.mark.parametrize("d", [1, 2, 4, 8])
@pytest.mark.parametrize("method", [0, 1])
def test_host_smoother_matches_the_oracle(host, d, method):
    T = 60
    P, S0, m0, B, Q, y = _wave_case(d, T, d)
    mask = np.ones(T, np.uint8)
    mask[[5, 17, 18]] = 0
    mean, cov = np.zeros((T, d), np.float32), np.zeros((T, d, d), np.float32)
    st = host.delta_host_smooth(d, method, T, _p(m0), _p(S0), _p(P), _p(B), _p(Q), _p(y),
                                mask.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)), _p(mean), _p(cov))
    assert st == 0
    sm, sc, _, _ = D.smooth_chain(y.astype(np.float64)[:, None], _wave(d), P, m0, S0,
                                  ("linearization", "unscented")[method], B=B.astype(np.float64), Q=Q, mask=mask)
    assert rel_l2(mean, sm) < TOL_MEAN and rel_l2(cov, sc) < TOL_COV, (rel_l2(mean, sm), rel_l2(cov, sc))


@pytest.mark.parametrize("d", [1, 2, 4, 8])
@pytest.mark.parametrize("method", [0, 1])
def test_host_vmp_step_matches_the_oracle(host, d, method):
    T, iters = 40, 5
    P, S0, m0, B, _, y = _wave_case(d, T, 10 + d)
    cm, cc, ct = m0.copy(), S0.copy(), np.array([1.0, 0.01], np.float32)
    mean, cov, tau = np.zeros((T, d), np.float32), np.zeros((T, d, d), np.float32), np.zeros((T, 2), np.float32)
    st = host.delta_host_vmp(d, method, T, iters, _p(P), _p(B), _p(y), _p(cm), _p(cc), _p(ct), _p(mean), _p(cov), _p(tau))
    assert st == 0
    om, oc, oa, ob = D.vmp_gamma_stream(y.astype(np.float64), _wave(d), P, B[0].astype(np.float64), m0, S0, 1.0, 0.01,
                                        iters, ("linearization", "unscented")[method])
    assert rel_l2(mean, om) < TOL_MEAN and rel_l2(cov, oc) < TOL_COV
    # the rate sums squared residuals (a second moment, fp32 under Linearization): the covariance tolerance
    assert rel_l2(tau[:, 0], oa) < TOL_MEAN and rel_l2(tau[:, 1], ob) < TOL_COV
    np.testing.assert_array_equal(cm, mean[-1])          # the carry is the last datum's q(x)
