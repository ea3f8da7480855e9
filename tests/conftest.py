import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_sessionstart(session):
    # torch's default of one intra-op thread per core makes the CPU oracle crawl on many-core hosts
    # (128 threads ran 60x slower than 16 on the GPU box): cap it for the whole test session
    import torch
    torch.set_num_threads(max(1, min(16, os.cpu_count() or 1)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "slow: multi-second CPU test")


@pytest.fixture(scope="session")
def hp():
    from whisper_vits_svc_b200 import hparams
    return hparams.load_hparams(os.path.join(ROOT, "configs", "base.yaml"))


@pytest.fixture(scope="session")
def sd(hp):
    from whisper_vits_svc_b200 import synth
    return synth.svc_state_dict(hp, 1234)
