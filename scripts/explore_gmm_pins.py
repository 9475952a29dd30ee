"""Exploration (not shipped, not imported): which reading of Distributions' `rand(rng, Categorical(p), n)` reproduces the
free-energy pins of gmm_univariate_tests.jl (284.76 +- 0.1, 10 iterations) and gmm_multivariate_tests.jl (3436.7 +- 0.1,
25 iterations)?  Data replayed with the restated StableRNG, prior / initial means of the multivariate test from
StableRNG(42) in the reference's draw order, every candidate label reading x every update order of the oracle.
Run from the repository root: python scripts/explore_gmm_pins.py"""
import sys

sys.path.insert(0, ".")
sys.path.insert(0, "tests")
from test_mixture import (CATEGORICAL_READINGS, PRIOR_KEYS, SCHEDULES, gaussian_mixture, multivariate_reference_data,  # noqa: E402
                          multivariate_reference_model, univariate_reference_data, univariate_reference_model)

_, _, ua = univariate_reference_model()
_, _, ma = multivariate_reference_model()
for reading in CATEGORICAL_READINGS:
    yu = univariate_reference_data(reading=reading)[0]
    ym = multivariate_reference_data(reading=reading)[0]
    for s in SCHEDULES:
        fu = gaussian_mixture(yu[:, None, None], *(ua[k] for k in PRIOR_KEYS), iterations=10, schedule=s)["free_energy"][-1, 0]
        fm = gaussian_mixture(ym[:, :, None], *(ma[k] for k in PRIOR_KEYS), iterations=25, schedule=s)["free_energy"][-1, 0]
        print(f"{reading:48s} {s:8s} univariate {fu:9.3f} (pin 284.76)   multivariate {fm:9.3f} (pin 3436.7)")
