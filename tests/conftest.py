import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100")
    from oracle.cpu_threads import tune_threads
    tune_threads(16)


@pytest.fixture(scope="session")
def tiny_cfg():
    from reazonspeech_b200.config import ModelConfig
    return ModelConfig.tiny()


@pytest.fixture(scope="session")
def tiny_sd(tiny_cfg):
    from reazonspeech_b200.weights import random_state_dict
    return random_state_dict(tiny_cfg, seed=0)


@pytest.fixture(scope="session")
def tiny_engine(tiny_cfg, tiny_sd):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from reazonspeech_b200.engine import Engine
    return Engine(tiny_cfg, tiny_sd, "cuda:0")
