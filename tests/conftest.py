import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN_DIR


def load_golden(name):
    import numpy as np

    return np.load(os.path.join(GOLDEN_DIR, f"mips_{name}.npz"), allow_pickle=False)


def golden_inputs(g):
    """Regenerate the inputs of a golden case and verify them against the stored sha256."""
    import synth

    n = int(g["n"])
    nq_per_rank = [int(x) for x in g["nq_per_rank"]]
    bank = synth.make_bank(n, seed=int(g["bank_seed"]), dist=str(g["dist"]))
    q = synth.make_queries(sum(nq_per_rank), seed=int(g["query_seed"]), dist=str(g["dist"]))
    assert synth.sha256(bank, q) == str(g["inputs_sha256"]), "synthetic inputs differ from the golden generator's"
    return bank, q, nq_per_rank
