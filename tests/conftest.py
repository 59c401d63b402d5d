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
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")
    config.addinivalue_line("markers", "multigpu: gpu test that spawns one process per GPU (needs >= 2 devices)")


def pytest_collection_modifyitems(config, items):
    """`gpu` tests need an H100: skip (not fail) them on a machine without CUDA; `multigpu` tests need >= 2 devices."""
    n = torch.cuda.device_count() if torch.cuda.is_available() else 0
    for item in items:
        if "gpu" in item.keywords and n == 0:
            item.add_marker(pytest.mark.skip(reason="no CUDA device (run on an H100 with -m gpu)"))
        elif "multigpu" in item.keywords and n < 2:
            item.add_marker(pytest.mark.skip(reason="needs >= 2 CUDA devices"))


def load_npz(name):
    z = np.load(os.path.join(GOLDEN, name), allow_pickle=False)
    return {k: (torch.from_numpy(z[k]) if z[k].dtype.kind in "fiub" and z[k].ndim > 0 else z[k]) for k in z.files}


def net_weights(z, prefix):
    """state-dict (reference key names, SURVEY A.1) of one FlexibleNeRFModel from a weights_*.npz."""
    p = prefix + "."
    return {k[len(p):]: v for k, v in z.items() if k.startswith(p)}


@pytest.fixture(scope="session")
def lego():
    z = load_npz("weights_lego_nerf.npz")
    return dict(coarse=net_weights(z, "coarse"), fine=net_weights(z, "fine"), u=z["sample_pdf_u"])


@pytest.fixture(scope="session")
def fern():
    z = load_npz("weights_fern_nerf.npz")
    return dict(coarse=net_weights(z, "coarse"), fine=net_weights(z, "fine"), u=z["sample_pdf_u"])


@pytest.fixture(scope="session")
def buff():
    z = load_npz("weights_lego_buff.npz")
    return dict(coarse=net_weights(z, "coarse"), voxels=z["voxels"])
