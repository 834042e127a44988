import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu)")


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session", autouse=True)
def _built():
    """The in-tree CUDA library must exist for every test session (the driver runs build() first)."""
    import __graft_entry__ as g
    g.build()


_PARITY = []


@pytest.fixture
def parity_log():
    """Record the margin a parity test measured (max / RMS |dz| on the decoder logit == relative depth error); the
    session writes them to gpurun_out/parity_margins.json (copied to profiles/PARITY_rNN.json per round)."""
    def log(case, against, dz, **extra):
        dz = dz.double().flatten()
        row = {"case": case, "against": against, "max_dz": float(dz.max()), "rms_dz": float(dz.pow(2).mean().sqrt()),
               "n": int(dz.numel()), "tolerance": 1e-3, **extra}
        _PARITY.append(row)
        print("\n[parity] " + " ".join(f"{k}={v:.3e}" if isinstance(v, float) else f"{k}={v}" for k, v in row.items()))
    return log


def pytest_sessionfinish(session, exitstatus):
    if not _PARITY:
        return
    import json
    out = os.path.join(ROOT, "gpurun_out")
    try:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "parity_margins.json"), "w") as f:
            json.dump({"metric": "|dz| on the decoder's pre-sigmoid logit (== relative depth error)", "rows": _PARITY}, f, indent=1)
    except OSError:
        pass
