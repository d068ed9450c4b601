"""pytest configuration: registers the `gpu` marker and builds the CPU oracle (test infrastructure)."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (run with -m gpu on an H100)")


@pytest.fixture(scope="session")
def oracle():
    from tests import oracle_lib

    return oracle_lib.load()


def pytest_sessionstart(session):
    # Debugging aid only: WTG_TEST_EMU=1 routes the C-ABI calls of the `-m gpu`
    # tests to the host-compiled build of the device logic (tests/emu) so that the *test logic* can be
    # exercised on a machine without a GPU.  Real parity runs happen on an H100 with this unset.
    if os.environ.get("WTG_TEST_EMU") == "1":
        from tests import emu_lib
        from wittgenstein_b200 import _lib

        _lib._api = emu_lib.api()
