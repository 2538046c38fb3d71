import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def pytest_collection_modifyitems(config, items):
    """`gpu`-marked tests are skipped (not errored) where the engine cannot run: no built library or no CUDA device.
    On a GPU box a missing library is still LOUD: tests/test_abi.py (CPU suite) fails when the .so is absent."""
    reason = None
    try:
        from pymc_b200 import _lib

        if not os.path.isfile(_lib.LIB_PATH):
            if os.path.exists("/dev/nvidiactl"):  # a GPU box without the built engine: fail loudly, do not skip
                return
            reason = f"{_lib.LIB_PATH} not built"
        elif _lib.load().b200_device_count() < 1:
            reason = "no CUDA device visible"
    except Exception as e:  # pragma: no cover
        reason = f"engine not loadable: {e}"
    if reason is None:
        return
    skip = pytest.mark.skip(reason=reason)
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def load_golden(name):
    d = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    if "z" not in d and "seeds" in d:
        # files kept under 1 MB store no momentum noise: it is the chain seed's own normal stream (oracle/make_golden.py)
        from oracle.make_golden import noise

        T = int(d["tune"]) + int(d["draws"])
        d["z"] = np.array([noise(int(s), T, d["q0"].shape[1]) for s in d["seeds"]])
    return d


@pytest.fixture(scope="session")
def golden():
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = load_golden(name)
        return cache[name]

    return get
