import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu)")


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="session")
def schema(golden_dir):
    import json
    with open(os.path.join(golden_dir, "state_dict_schema.json")) as f:
        return json.load(f)


@pytest.fixture(scope="session")
def synth_sd(schema):
    from oracle import weights as W
    return W.synth_state_dict([(n, tuple(s)) for n, s in schema["entries"]])
