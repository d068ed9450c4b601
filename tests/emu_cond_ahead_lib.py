"""TEST INFRASTRUCTURE — loads the host build of the device logic (tests/emu) with the pass shapes of an unsharded GSF network
whose next checkSigs runs ahead (tests/emu/wtg_emu_cond_ahead.cpp).  Every other network behaves as in tests/emu_lib.py.
Never used by the product package."""
import os
import subprocess

from tests.emu_lib import EMU_DIR, ROOT
from wittgenstein_b200 import _lib

_api = None


def api():
    global _api
    if _api is not None:
        return _api
    so = os.path.join(EMU_DIR, "libwtg_emu_cond_ahead.so")
    src = os.path.join(EMU_DIR, "wtg_emu_cond_ahead.cpp")
    csrc = os.path.join(ROOT, "wittgenstein_b200", "csrc")
    srcs = [src, os.path.join(EMU_DIR, "wtg_emu.cpp")] + [os.path.join(csrc, f) for f in os.listdir(csrc)]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        tmp = f"{so}.{os.getpid()}.tmp"  # concurrent test workers: each links its own file, the rename is atomic
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", tmp, src])
        os.replace(tmp, so)
    _api = _lib.Api(so, "wtgemuc_")
    return _api
