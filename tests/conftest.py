import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")
    config.addinivalue_line("markers", "slow: full-size CPU checks (seconds each)")


@pytest.fixture(scope="session")
def golden():
    import json
    return json.loads((ROOT / "tests" / "golden" / "golden.json").read_text())
