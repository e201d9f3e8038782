import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a); run with -m gpu")


@pytest.fixture(scope="session")
def w2l_state_dict():
    """Seeded conditioned synthetic wav2lip256 weights (oracle.wav2lip_ref.synth_state_dict(0)), cached on disk."""
    import torch
    from oracle import wav2lip_ref as R
    cache = os.path.join("/tmp", "ltb_w2l_sd_seed0.pt")
    if os.path.exists(cache):
        try:
            return torch.load(cache)
        except Exception:
            pass
    sd = R.synth_state_dict(0)
    try:
        torch.save(sd, cache)
    except Exception:
        pass
    return sd


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN
