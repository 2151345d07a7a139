import os
import sys
import warnings

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

warnings.filterwarnings("ignore")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


def pytest_collection_modifyitems(config, items):
    # plain `pytest tests` on a box without a CUDA device: the gpu tests are skipped (they would all raise "no CUDA device
    # visible" and bury real failures of the CPU suite).  An explicit `-m gpu` still runs them, so that a GPU box whose device
    # went missing fails loudly instead of passing with everything skipped.
    markexpr = config.getoption("markexpr", "") or ""
    asked_for_gpu = "gpu" in markexpr and "not gpu" not in markexpr
    skip_gpu = None
    if not asked_for_gpu:
        try:
            import torch
            have_cuda = torch.cuda.is_available()
        except Exception:                                   # noqa: BLE001
            have_cuda = False
        if not have_cuda:
            skip_gpu = pytest.mark.skip(reason="no CUDA device visible (run with -m gpu on an H100)")
    for item in items:
        if skip_gpu is not None and "gpu" in item.keywords:
            item.add_marker(skip_gpu)


@pytest.fixture(scope="session")
def syn_model():
    from mvsmplfitting_b200 import synthetic as S
    return S.make_model(0)


@pytest.fixture(scope="session")
def syn_gmm():
    from mvsmplfitting_b200 import synthetic as S
    return S.make_gmm(7)
