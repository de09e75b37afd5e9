import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def pytest_sessionstart(session):
    # the oracle runs on the host: on a large shared host, a hundred-odd threads make torch CPU ops much slower than
    # 8-16 threads do; keep the CPU side of the tests predictable
    import torch
    torch.set_num_threads(min(16, os.cpu_count() or 1))


def pytest_terminal_summary(terminalreporter, exitstatus, config):
    # how much of the parity rests on the S8(c) escape hatch (tests/parity_util.py)
    try:
        from tests import parity_util
        parity_util.report(terminalreporter.write_line)
    except Exception:
        pass
