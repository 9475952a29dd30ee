"""Delta-node test models: CUDA sources for the library and the matching fp64 callables (with analytic Jacobians) for
oracle/delta.py."""
import numpy as np

from oracle import delta as D

PENDULUM_SRC = """
template <class S> __device__ void pendulum(const S* x, S* z) {
    const double dt = 0.01, G = 9.81;
    z[0] = x[0] + x[1] * dt;
    z[1] = x[1] - G * sin(x[0]) * dt;
}
"""

# constant-velocity target (dt = 0.1) observed by range and bearing from a sensor at (-3, -2)
TRACKER_SRC = """
template <class S> __device__ void cv(const S* x, S* z) {
    const double dt = 0.1;
    z[0] = x[0] + dt * x[2]; z[1] = x[1] + dt * x[3]; z[2] = x[2]; z[3] = x[3];
}
template <class S> __device__ void range_bearing(const S* x, S* y) {
    const S dx = x[0] + 3.0, dy = x[1] + 2.0;
    y[0] = sqrt(dx * dx + dy * dy);
    y[1] = atan2(dy, dx);
}
"""


def _cv(x):
    return np.array([x[0] + 0.1 * x[2], x[1] + 0.1 * x[3], x[2], x[3]])


def _rb(x):
    dx, dy = x[0] + 3.0, x[1] + 2.0
    return np.array([np.hypot(dx, dy), np.arctan2(dy, dx)])


def _rb_jac(x):
    dx, dy = x[0] + 3.0, x[1] + 2.0
    r2 = dx * dx + dy * dy
    r = np.sqrt(r2)
    return np.array([[dx / r, dy / r, 0, 0], [-dy / r2, dx / r2, 0, 0]])


CV_A = np.array([[1, 0, 0.1, 0], [0, 1, 0, 0.1], [0, 0, 1, 0], [0, 0, 0, 1.0]])
TRACKER_F = D.Fn(_cv, lambda x: CV_A)
TRACKER_G = D.Fn(_rb, _rb_jac)

# d = 8: a mildly nonlinear coupled map, observed in 3 components through a quadratic g
D8_SRC = """
template <class S> __device__ void f8(const S* x, S* z) {
    for (int i = 0; i < 8; ++i) z[i] = 0.9 * x[i] + 0.1 * tanh(x[(i + 1) % 8]);
}
template <class S> __device__ void g8(const S* x, S* y) {
    for (int k = 0; k < 3; ++k) y[k] = x[k] + 0.05 * x[k + 3] * x[k + 3];
}
"""


def _f8(x):
    return 0.9 * x + 0.1 * np.tanh(np.roll(x, -1))


def _f8_jac(x):
    J = 0.9 * np.eye(8)
    for i in range(8):
        J[i, (i + 1) % 8] += 0.1 * (1 - np.tanh(x[(i + 1) % 8]) ** 2)
    return J


def _g8(x):
    return x[:3] + 0.05 * x[3:6] ** 2


def _g8_jac(x):
    J = np.zeros((3, 8))
    for k in range(3):
        J[k, k] = 1.0
        J[k, k + 3] = 0.1 * x[k + 3]
    return J


D8_F = D.Fn(_f8, _f8_jac)
D8_G = D.Fn(_g8, _g8_jac)


def simulate(f, g, B, P, Q, m0, S0, T, batch, seed):
    """y[T, m, batch] drawn from x[1] ~ N(m0, S0), x[t] = f(x[t-1]) + N(0, P), y ~ N(g(x) or B x, Q)."""
    rng = np.random.default_rng(seed)
    d = len(m0)
    LP, LQ, LS = (np.linalg.cholesky(M) for M in (P, Q, S0))
    m = Q.shape[0]
    y = np.zeros((T, m, batch))
    for b in range(batch):
        x = m0 + LS @ rng.standard_normal(d)
        for t in range(T):
            if t > 0:
                x = f.h(x) + LP @ rng.standard_normal(d)
            y[t, :, b] = (g.h(x) if g is not None else B @ x) + LQ @ rng.standard_normal(m)
    return y
