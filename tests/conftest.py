import os
import sys

# Several contexts (= "ranks") with their own streams share one process in tests/test_peer_gather_gpu.py; with the default
# 8 hardware work queues their streams can alias, and a kernel queued behind another rank's spinning barrier kernel would
# never start.  Must be set before the CUDA context exists.  (Real multi-GPU jobs run one process per GPU.)
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
# (Same single-process caveat for CUDA lazy loading: the FIRST launch of a kernel loads its module, which can wait for
# running kernels; rxg_peer_group therefore loads the gather kernels up front, and the tests below run every sweep once
# without a gather -- the reference result -- before the virtual ranks gather.)

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def rx():
    import rxinfer_jl_b200
    return rxinfer_jl_b200


@pytest.fixture(scope="session")
def ctx(rx):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return rx.Context(0)


_OPTION_DEFAULTS = {"gain_seq": 0, "large_seq": 0, "no_umma": 0, "sweep_variant": 0, "force_cpt": 0, "host_threads": 0,
                    "host_cov_d2h": 0, "host_bcast_min_mb": 64, "host_slices": 0, "gather_mode": 0}


@pytest.fixture(autouse=True)
def _reset_ctx_options(request):
    """The ctx is session scoped; tests flip dispatch options (ctx.set_option) and must not leak them."""
    yield
    if "ctx" in request.fixturenames:
        try:
            c = request.getfixturevalue("ctx")
        except Exception:
            return
        for k, v in _OPTION_DEFAULTS.items():
            c.set_option(k, v)
