"""grp_batch_schedule against the reference's GrpFileDatasetsIter + DataLoader(batch_size, drop_last=True), restated over stub
per-file game lengths: the same batches of the same prefixes, and the same `random` state afterwards, for cycle=False and
cycle=True, batch sizes below and above a file batch's buffer, and empty file batches."""
import random

import numpy as np
import pytest

import grp_train_lib as T
from mortal_b200.grp_train import grp_batch_schedule


def stub_files(n_files, rng, empty_every=0):
    """file name -> list of game lengths (a file with no games when empty_every divides its index)"""
    return {f"f{i:03d}": ([] if empty_every and i % empty_every == 0 else [int(x) for x in rng.integers(1, 13, size=rng.integers(1, 3))])
            for i in range(n_files)}


def reference(files, file_batch_size, cycle, batch_size, n_batches):
    """the restated reference: each sample as (file, game, prefix length)"""
    names = list(files)

    def load(chunk):  # a kyoku row encodes (file index, game); the prefix length is the sample's row count
        return [(np.array([[names.index(name), g, k, 0, 0, 0, 0] for k in range(n)], dtype=np.float64), None)
                for name in chunk for g, n in enumerate(files[name])]

    it = T.RefGrpFileDatasetsIter(list(files), load, file_batch_size, cycle)
    return [[(names[int(x[-1, 0])], int(x[-1, 1]), len(x)) for x, _ in b] for b in T.ref_batches(it, batch_size, n_batches)]


def ours(files, file_batch_size, cycle, batch_size, n_batches):
    file_list = list(files)
    samples = []

    def cycle_sizes():
        random.shuffle(file_list)
        for start in range(0, len(file_list), file_batch_size):
            n = 0
            for name in file_list[start:start + file_batch_size]:
                for g, m in enumerate(files[name]):
                    samples.extend((name, g, k + 1) for k in range(m))
                    n += m
            yield n

    def passes():
        while True:
            yield cycle_sizes()
            if not cycle:
                break

    out = []
    for ids in grp_batch_schedule(passes(), batch_size):
        out.append([samples[i] for i in ids])
        if n_batches is not None and len(out) == n_batches:
            break
    return out


@pytest.mark.parametrize("cycle", [False, True])
@pytest.mark.parametrize("batch_size", [1, 7, 64, 500])
@pytest.mark.parametrize("empty_every", [0, 3])
def test_schedule_matches_reference(cycle, batch_size, empty_every):
    files = stub_files(23, np.random.default_rng(batch_size + empty_every), empty_every)
    n_batches = 40 if cycle else None
    random.seed(1234)
    want = reference(files, 5, cycle, batch_size, n_batches)
    state = random.getstate()
    random.seed(1234)
    got = ours(files, 5, cycle, batch_size, n_batches)
    assert got == want
    assert random.getstate() == state
    assert want or (not cycle and batch_size == 500)


def test_every_file_batch_empty():
    files = {f"f{i}": [] for i in range(4)}
    random.seed(5)
    want = reference(files, 2, False, 3, None)
    state = random.getstate()
    random.seed(5)
    assert ours(files, 2, False, 3, None) == want == []
    assert random.getstate() == state


def test_bad_batch_size():
    with pytest.raises(ValueError):
        list(grp_batch_schedule([[3]], 0))
