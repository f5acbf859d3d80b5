import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def port():
    from oracle.oracle import Port
    return Port()


def _rand2k(path):
    """rand2k.npz stores the seeded l2 / ip table (make_golden.py: default_rng(42)) as a CRC only; it is redrawn here."""
    import zlib
    import numpy as np
    g = dict(np.load(path, allow_pickle=False))
    X = np.random.default_rng(42).random((2300, 32), dtype=np.float32)
    assert zlib.crc32(X.tobytes()) == int(g["table_crc32"]), "numpy no longer draws the rand2k table"
    g["stored_l2"] = g["stored_ip"] = X
    return g


@pytest.fixture(scope="session")
def golden():
    import numpy as np
    d = os.path.join(ROOT, "tests", "golden")
    out = {n: np.load(os.path.join(d, n + ".npz"), allow_pickle=False) for n in ("dense_vector", "halfcircle")}
    out["rand2k"] = _rand2k(os.path.join(d, "rand2k.npz"))
    return out


@pytest.fixture(scope="session")
def have_ref():
    from oracle import oracle
    return oracle.have_ref()


@pytest.fixture(scope="session")
def golden_refgraph():
    import numpy as np
    return np.load(os.path.join(ROOT, "tests", "golden", "refgraph20k.npz"), allow_pickle=False)
