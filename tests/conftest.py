import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "oracle"), os.path.join(ROOT, "img2img-turbo_b200"), ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)


import torch
torch.set_num_threads(min(32, os.cpu_count() or 1))     # many-core GPU hosts run the CPU oracle faster without every thread


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a GPU host)")


@pytest.fixture(scope="session")
def tiny_sd():
    import weights as W
    return W.make_state_dict("pix2pix", W.TINY, seed=0, perturb_norm=True)


@pytest.fixture(scope="session")
def tiny_sd_cyc():
    import weights as W
    return W.make_state_dict("cyclegan", W.TINY, seed=0, perturb_norm=True)
