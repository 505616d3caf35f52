import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)
sys.dont_write_bytecode = True


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (sm_90)")
