import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")


def _ensure_native_artifacts():
    """A fresh checkout has no built artefacts (they are git-ignored): build them once (nvcc cross-compiles
    without a GPU).  Tests never fall back to anything else if this fails."""
    lib = os.path.join(ROOT, "distributed_cluster_gpus_b200", "csrc", "libdcsim_b200.so")
    srcs = [os.path.join(ROOT, "distributed_cluster_gpus_b200", "csrc", f)
            for f in ("dcsim_b200.cu", "dcsim_core.cuh", "dcsim_advance_impl.cuh", "dcsim_advance_g8.cu", "dcsim_advance_g16.cu")]
    stale = (not os.path.exists(lib)) or any(os.path.getmtime(s) > os.path.getmtime(lib) for s in srcs)
    if stale:
        import __graft_entry__
        __graft_entry__.build()


_ensure_native_artifacts()


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a)")


def golden_names():
    return sorted(f[:-5] for f in os.listdir(GOLDEN_DIR) if f.endswith(".json") and f not in ("kat.json", "fuzz_reference.json", "ill_conditioned_cap_greedy_case.json",
                                                                                   "ill_conditioned_cap_greedy_cases_r2.json"))


def load_fuzz_reference():
    """Random scenarios run through the unmodified reference (tests/golden/make_golden_fuzz.py)."""
    with open(os.path.join(GOLDEN_DIR, "fuzz_reference.json")) as f:
        return json.load(f)["cases"]


def load_golden(name):
    with open(os.path.join(GOLDEN_DIR, name + ".json")) as f:
        return json.load(f)


@pytest.fixture(scope="session")
def oracle():
    import oracle_lib
    oracle_lib.build()
    return oracle_lib


@pytest.fixture(scope="session")
def hostemu():
    import hostemu_lib
    hostemu_lib.lib()
    return hostemu_lib


def has_cuda():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False
