"""bench.py --dump-outputs: the arrays a caller of the timed path reads back are written as float64 / float32 .npy files, never
more than DUMP_MAX_BYTES; per-node arrays that do not fit are written for a fixed, seeded sample of the nodes.  CPU only: the
protocol objects are stand-ins with the read-back methods of wittgenstein_b200.GSFSignature / CasperIMD."""
import os

import numpy as np
import pytest

import bench


class _Net:
    def __init__(self, n):
        self.n = n

    def counters(self):
        return np.arange(5 * self.n, dtype=np.int64).reshape(5, self.n)


class _GSF:
    def __init__(self, n, levels, words):
        self.n, self.levels, self.words = n, levels, words

    def network(self):
        return _Net(self.n)

    def scalars(self):
        return {"card": np.arange(self.n, dtype=np.int32), "pairing": np.full(self.n, 4, np.int32)}

    def level_scalars(self):
        return {"pos": np.arange(self.n * self.levels, dtype=np.int32).reshape(self.n, self.levels)}

    def verified(self):
        return np.full((self.n, self.words), 0x8000000000000001, np.uint64)


class _Casper:
    def __init__(self, n, blocks):
        self.n, self.nb = n, blocks

    def network(self):
        return _Net(self.n)

    def node_state(self):
        return {"head": np.arange(self.n, dtype=np.int32) % self.nb, "hs": np.arange(self.n, dtype=np.uint64) * np.uint64(0x100000003)}

    def heads(self):
        return np.arange(self.n, dtype=np.int32) % self.nb

    def blocks(self):
        return {"height": np.arange(self.nb, dtype=np.int32), "parent": np.arange(self.nb, dtype=np.int32) - 1}


def _load(d):
    return {f[:-4]: np.load(os.path.join(d, f)) for f in os.listdir(d)}


def _check_common(files):
    assert sum(a.nbytes for a in files.values()) <= bench.DUMP_MAX_BYTES
    assert all(a.dtype in (np.float32, np.float64) for a in files.values())


@pytest.mark.parametrize("n, levels, words, sampled", [(1024, 4, 16, False), (1 << 17, 96, 8, True)])
def test_dump_outputs_gsf(tmp_path, n, levels, words, sampled):
    bench.dump_outputs(str(tmp_path / "a"), *bench.gsf_outputs(_GSF(n, levels, words)))
    files = _load(tmp_path / "a")
    _check_common(files)
    nodes = files["nodes"].astype(np.int64)
    assert (len(nodes) < n) == sampled and (np.diff(nodes) > 0).all() and nodes[-1] < n
    assert (files["scalar_card"] == nodes).all()
    assert (files["counters"][1] == n + nodes).all()
    assert (files["level_pos"][:, 1] == nodes * levels + 1).all()
    rows = files["verified_rows"]
    assert rows.shape == (bench.DUMP_ROWS, words * 64) and (rows[:, 0] == 1).all() and (rows[:, 63] == 1).all() and rows[:, 1:63].sum() == 0
    bench.dump_outputs(str(tmp_path / "b"), *bench.gsf_outputs(_GSF(n, levels, words)))
    again = _load(tmp_path / "b")
    assert again.keys() == files.keys() and all((again[k] == v).all() for k, v in files.items())


def test_dump_outputs_gsf_rows_fit_the_budget(tmp_path):
    words = bench.DUMP_MAX_BYTES // 4 // (64 * 4) // 8 * 2  # one row is a quarter of the budget / 4: four rows fit
    bench.dump_outputs(str(tmp_path), *bench.gsf_outputs(_GSF(64, 2, words)))
    files = _load(tmp_path)
    _check_common(files)
    assert files["verified_rows"].shape[0] == 4 and len(files["nodes"]) == 64


def test_dump_outputs_casper(tmp_path):
    n, nb = 1000, 7
    bench.dump_outputs(str(tmp_path), *bench.casper_outputs(_Casper(n, nb)))
    files = _load(tmp_path)
    _check_common(files)
    hs = np.arange(n, dtype=np.uint64) * np.uint64(0x100000003)
    assert (files["node_hs_lo32"] == (hs & np.uint64(0xFFFFFFFF)).astype(np.float64)).all()
    assert (files["node_hs_hi32"] == (hs >> np.uint64(32)).astype(np.float64)).all()
    assert (files["node_head"] == np.arange(n) % nb).all() and (files["heads"] == files["node_head"]).all()
    assert files["counters"].shape == (5, n) and (files["block_parent"] == np.arange(nb) - 1).all()
    assert len(files["nodes"]) == n
