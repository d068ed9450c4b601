"""__graft_entry__.build() rebuilds the CUDA library when it is missing, older than a source, or was built with other nvcc
flags (a library left over from a build for another architecture must not be kept).  CPU only: checks the staleness rule."""
import os

import __graft_entry__ as g


def test_stale_when_flags_differ_or_are_unrecorded(tmp_path):
    src = tmp_path / "k.cu"
    so = tmp_path / "lib.so"
    src.write_text("")
    so.write_text("")
    os.utime(src, (1000, 1000))
    os.utime(so, (2000, 2000))
    flags = ["-gencode", "arch=compute_90a,code=sm_90a"]
    assert g._stale(str(so), [str(src)], flags)  # no record of the flags
    (tmp_path / "lib.so.flags").write_text(" ".join(flags))
    assert not g._stale(str(so), [str(src)], flags)
    assert g._stale(str(so), [str(src)], ["-gencode", "arch=compute_100a,code=sm_100a"])
    os.utime(src, (3000, 3000))
    assert g._stale(str(so), [str(src)], flags)
    assert g._stale(str(tmp_path / "missing.so"), [str(src)], flags)
