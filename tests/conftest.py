import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a)")
    # The CPU oracle legs: torch's default of one thread per host CPU oversubscribes the small GEMMs of the checker on
    # many-core hosts and roughly doubles the time of the GPU suite.  The cap changes nothing about the results.
    torch.set_num_threads(max(1, min(32, os.cpu_count() or 1)))


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


def load_golden(name):
    with np.load(os.path.join(GOLDEN, name + ".npz")) as z:
        return {k: torch.from_numpy(z[k]) for k in z.files}


@pytest.fixture(scope="session")
def golden():
    return load_golden


@pytest.fixture(scope="session")
def weights_cpu():
    """Seeded oracle weights (reference-free; identical on every machine)."""
    from oracle import weights
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = dict(g=weights.g_state_dict, plm=weights.plm_state_dict, adm=weights.adm_state_dict,
                               hifigan=weights.hifigan_state_dict)[name]()
        return cache[name]
    return get
