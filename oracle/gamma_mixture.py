"""fp64 restatement of mean-field VMP for the Gamma mixture model with point-mass shapes (GammaMixture node;
DESIGN 3.24; ref: test/models/mixtures/gamma_mixture_tests.jl:7-40).

    s ~ Dirichlet(α_s);  a[k] ~ Gamma(α_a[k], β_a[k]);  b[k] ~ Gamma(α_b[k], β_b[k])   (shape, rate)
    z[i] ~ Categorical(s);  y[i] ~ GammaMixture(switch = z[i], a = a, b = b)   (component k: Gamma(shape a[k], rate b[k]))
    q(z) q(a) q(b) q(s),  q(a[k]) = PointMass(â_k)

With r_ik = q(z_i = k), N_k = Σ_i r_ik, S_k = Σ_i r_ik y_i, L_k = Σ_i r_ik log y_i each update is the exact coordinate
minimiser of the free energy F (``free_energy``):
    a: â_k = argmax (α_a − 1) log a − β_a a + a (N_k E[log b_k] + L_k) − N_k lgamma(a)   (``point_mass_shape``)
    b: q(b_k) = Gamma(α_b + â_k N_k, β_b + S_k)
    s: q(s) = Dirichlet(α_s + N)
    z: q(z_i) ∝ exp(E[log s_k] + â_k E[log b_k] − lgamma(â_k) + (â_k − 1) log y_i − E[b_k] y_i)
``gamma_mixture(..., schedule=)`` runs them in any order per iteration; the library runs "absz".  Arrays of ``batch``
independent data sets: y [N, batch]; hyper-parameters [K], shared."""
import numpy as np
from scipy.special import digamma, gammaln, polygamma

NEWTON_CAP = 100
NEWTON_RTOL = 1e-12


def point_mass_shape(ash, art, n, c, a0):
    """The maximiser of f(a) = (ash − 1) log a − art a + a c − n lgamma(a) by Newton's method from a0, elementwise; an
    iterate that would leave a > 0 is replaced by half the current one.  Returns (a, converged)."""
    ash, art, n, c = np.broadcast_arrays(*(np.asarray(x, np.float64) for x in (ash, art, n, c)))
    a = np.broadcast_to(np.asarray(a0, np.float64), n.shape).copy()
    done = np.zeros(n.shape, bool)
    for _ in range(NEWTON_CAP):
        g = (ash - 1.0) / a - art + c - n * digamma(a)
        h = -(ash - 1.0) / (a * a) - n * polygamma(1, a)
        with np.errstate(divide="ignore", invalid="ignore"):
            an = a - g / h
        an = np.where(an > 0.0, an, 0.5 * a)
        step = np.abs(an - a) <= NEWTON_RTOL * an
        a = np.where(done, a, an)
        done |= step
        if done.all():
            break
    return a, done


def kl_gamma(a1, b1, a0, b0):
    """KL(Gamma(a1, b1) || Gamma(a0, b0)), shape / rate."""
    return (a1 - a0) * digamma(a1) - gammaln(a1) + gammaln(a0) + a0 * (np.log(b1) - np.log(b0)) + a1 * (b0 - b1) / b1


def kl_dirichlet(al, al0):
    """KL(Dirichlet(al) || Dirichlet(al0)) over axis 0."""
    sa = al.sum(0)
    return (gammaln(sa) - gammaln(al).sum(0) - gammaln(al0.sum(0)) + gammaln(al0).sum(0)
            + ((al - al0) * (digamma(al) - digamma(sa))).sum(0))


def log_rho(y, alpha, a, bsh, brt):
    """log of the unnormalised q(z): [N, K, batch]."""
    els = digamma(alpha) - digamma(alpha.sum(0))
    elb = digamma(bsh) - np.log(brt)
    ly = np.log(y)[:, None]
    return (els + a * elb - gammaln(a))[None] + (a - 1.0)[None] * ly - (bsh / brt)[None] * y[:, None]


def statistics(y, r):
    return r.sum(0), (r * y[:, None]).sum(0), (r * np.log(y)[:, None]).sum(0)


def free_energy(y, r, alpha, a, bsh, brt, prior):
    """F at q(z) = r [N, K, batch], q(s) = Dirichlet(alpha), â = a, q(b) = Gamma(bsh, brt) (the point masses' entropy
    left out, their prior evaluated at the point), from the sufficient statistics."""
    Nk, Sk, Lk = statistics(y, r)
    als, ash, art, bsh0, brt0 = (np.asarray(prior[k], np.float64)[:, None] for k in
                                 ("alpha_s", "a_shape0", "a_rate0", "b_shape0", "b_rate0"))
    els = digamma(alpha) - digamma(alpha.sum(0))
    elb = digamma(bsh) - np.log(brt)
    logp_a = ash * np.log(art) - gammaln(ash) + (ash - 1.0) * np.log(a) - art * a
    with np.errstate(divide="ignore", invalid="ignore"):
        ent = -np.where(r > 0, r * np.log(r), 0.0).sum((0, 1))
    return (kl_dirichlet(alpha, np.broadcast_to(als, alpha.shape)) + kl_gamma(bsh, brt, bsh0, brt0).sum(0)
            - logp_a.sum(0)
            - (Nk * els + a * Nk * elb - Nk * gammaln(a) + (a - 1.0) * Lk - bsh / brt * Sk).sum(0) - ent)


def gamma_mixture(y, alpha_s, a_shape0, a_rate0, b_shape0, b_rate0, alpha_init, b_shape_init, b_rate_init, a_start,
                  iterations=10, schedule="absz"):
    """Mean-field VMP over y [N, batch] from a uniform q(z), q(s) = Dirichlet(alpha_init), q(b) = Gamma(b_shape_init,
    b_rate_init) and â = a_start, the updates of each iteration in the order of ``schedule`` (a permutation of "absz").
    Returns the last marginals (``alpha``, ``a_hat``, ``b_shape``, ``b_rate``, ``z_prob``), the histories ``hist_a``,
    ``hist_b_shape``, ``hist_b_rate`` [iterations, K, batch], ``free_energy`` [iterations, batch] and ``converged``
    [batch] (every Newton iteration converged)."""
    assert sorted(schedule) == sorted("absz"), schedule
    y = np.asarray(y, np.float64)
    N, nb = y.shape
    prior = dict(alpha_s=alpha_s, a_shape0=a_shape0, a_rate0=a_rate0, b_shape0=b_shape0, b_rate0=b_rate0)
    col = lambda v: np.repeat(np.asarray(v, np.float64)[:, None], nb, 1)
    K = len(alpha_s)
    r = np.full((N, K, nb), 1.0 / K)
    alpha, bsh, brt, a = col(alpha_init), col(b_shape_init), col(b_rate_init), col(a_start)
    conv = np.ones(nb, bool)
    hist = {k: np.zeros((iterations, K, nb)) for k in ("hist_a", "hist_b_shape", "hist_b_rate")}
    fe = np.zeros((iterations, nb))
    for it in range(iterations):
        for u in schedule:
            Nk, Sk, Lk = statistics(y, r)
            if u == "a":
                a, ok = point_mass_shape(col(a_shape0), col(a_rate0), Nk, Nk * (digamma(bsh) - np.log(brt)) + Lk,
                                         col(a_start))
                conv &= ok.all(0)
            elif u == "b":
                bsh, brt = col(b_shape0) + a * Nk, col(b_rate0) + Sk
            elif u == "s":
                alpha = col(alpha_s) + Nk
            else:
                lr = log_rho(y, alpha, a, bsh, brt)
                lr -= lr.max(1, keepdims=True)
                r = np.exp(lr)
                r /= r.sum(1, keepdims=True)
        hist["hist_a"][it], hist["hist_b_shape"][it], hist["hist_b_rate"][it] = a, bsh, brt
        fe[it] = free_energy(y, r, alpha, a, bsh, brt, prior)
    return dict(alpha=alpha, a_hat=a, b_shape=bsh, b_rate=brt, z_prob=r, free_energy=fe, converged=conv, **hist)
