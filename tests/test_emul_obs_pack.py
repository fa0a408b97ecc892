"""The training-buffer observation codec (csrc/mjx_obs_pack.cuh, host build): records of every obs version and of the invisible
observation round-trip bit for bit through unpack for any gather, every row outside the value-row table is 0 / 1 in real
observations, the record sizes are those of the layout, and a mask row with any other bit pattern is refused with the sample's
first such row, never rounded into the mask."""
import numpy as np
import pytest

import obs_pack_lib as P
import oracle_lib as O
import validate_lib as VL

SIZES = {(1, False): 8184, (2, False): 16104, (3, False): 17400, (4, False): 19112, (1, True): 1688, (2, True): 2144,
         (3, True): 2144, (4, True): 2144}


@pytest.fixture(scope="module")
def observations():
    """(version, invisible) -> float32 [n, rows, 34]: self-play decisions of run_sample_obs (with their invisible observations),
    plus every move of the golden game and of self-play logs through gameplay_load (kan selections included, v4 with the
    single-player block)"""
    games = [P.golden_events()] + VL.emul_games(3, 1, seed0=8100)
    out = {}
    for v in (1, 2, 3, 4):
        obs, inv = P.sample_obs(v)
        obs_l, inv_l = [obs], [inv]
        for g in games:
            for p in range(4):
                r = O.gameplay_load(g, p, version=v, sp_mode=1, oracle_seed=tuple(g[0].get("seed", (0, 0))))
                obs_l.append(r["obs"]); inv_l.append(r["invisible"])
        out[v, False] = np.concatenate(obs_l)
        out[v, True] = np.concatenate(inv_l)
    return out


def _bits(x):
    return np.ascontiguousarray(x).view(np.int32)


@pytest.mark.parametrize("version,invisible", sorted(SIZES))
def test_record_bytes(version, invisible):
    assert P.record_bytes(version, invisible) == SIZES[version, invisible]
    rows, vals = P.ROWS[version, invisible], P.value_rows(version, invisible)
    assert SIZES[version, invisible] == rows * 8 + len(vals) * 136
    assert (np.diff(vals) > 0).all() and vals.min(initial=0) >= 0 and vals.max(initial=0) < rows
    assert P.record_bytes(0, 0) == -2 and P.record_bytes(5, 0) == -2 and P.record_bytes(4, 2) == -2


def test_value_rows_of_v4_and_invisible():
    v4 = set(P.value_rows(4, False).tolist())
    assert {889, 890} | set(range(961, 1012)) <= v4 and not (set(range(891, 961)) & v4) and len(v4) == 81
    assert P.value_rows(2, True).tolist() == [14, 31, 48] and len(P.value_rows(1, True)) == 0


@pytest.mark.parametrize("version,invisible", sorted(SIZES))
def test_round_trip(observations, version, invisible):
    x = observations[version, invisible]
    assert len(x) > 200
    vals = P.value_rows(version, invisible)
    mask_rows = np.setdiff1d(np.arange(x.shape[1]), vals)
    cells = _bits(x[:, mask_rows])
    assert np.isin(cells, [0, 0x3F800000]).all()  # every row outside the value table is 0 / 1 in every sample
    if version == 4 and not invisible:
        assert (x[:, 889:1012] != 0).any(axis=(1, 2)).sum() > 10  # the single-player block is exercised
    rc, rec, status = P.pack(x, version, invisible)
    assert rc == 0 and not status.any()
    rc, y = P.unpack(rec, np.arange(len(x)), version, invisible)
    assert rc == 0 and np.array_equal(_bits(y), _bits(x))
    rng = np.random.default_rng(version + 10 * invisible)
    perm = rng.integers(0, len(x), size=3 * len(x) // 2)  # a gather with repeats
    rc, y = P.unpack(rec, perm, version, invisible)
    assert rc == 0 and np.array_equal(_bits(y), _bits(x[perm]))


@pytest.mark.parametrize("version,invisible", [(4, False), (2, False), (1, False), (4, True), (1, True)])
def test_hostile_mask_cells(observations, version, invisible):
    """0.5, -0.0, NaN, 2.0 and denormals in a mask row give the sample's status 1 + the first such row"""
    x = observations[version, invisible][:40].copy()
    vals = set(P.value_rows(version, invisible).tolist())
    mask_rows = [r for r in range(x.shape[1]) if r not in vals]
    rng = np.random.default_rng(7)
    hostile = np.array([0.5, -0.0, np.nan, 2.0, np.float32(1e-45), np.float32(-1e-40), np.inf, 1.0000001], dtype=np.float32)
    want = np.zeros(len(x), dtype=np.int32)
    for i in range(0, len(x), 2):
        rows = sorted(rng.choice(mask_rows, size=int(rng.integers(1, 4)), replace=False))
        for r in rows:
            x[i, r, int(rng.integers(0, 34))] = hostile[(i // 2) % len(hostile)]
        want[i] = rows[0] + 1
    x[1, mask_rows[-1], 33] = np.float32(-0.0)  # the last cell of the last mask row
    want[1] = mask_rows[-1] + 1
    rc, rec, status = P.pack(x, version, invisible)
    assert rc == 0 and np.array_equal(status, want)


@pytest.mark.parametrize("version,invisible", [(4, False), (3, False), (2, True)])
def test_value_rows_keep_any_bits(observations, version, invisible):
    x = observations[version, invisible][:30].copy()
    vals = P.value_rows(version, invisible)
    rng = np.random.default_rng(11)
    b = x.view(np.uint32)
    b[:, vals] = rng.integers(0, 2**32, size=(len(x), len(vals), 34), dtype=np.uint32)  # NaN payloads, -0.0, denormals, ...
    b[0, vals, :4] = [0x7FC00001, 0xFF800000, 0x80000000, 0x00000001]
    rc, rec, status = P.pack(x, version, invisible)
    assert rc == 0 and not status.any()
    rc, y = P.unpack(rec, np.arange(len(x))[::-1], version, invisible)
    assert rc == 0 and np.array_equal(_bits(y), _bits(x[::-1]))


def test_pitch_reads_a_slice_in_place(observations):
    """a sample pitch larger than one observation reads every other sample of a buffer"""
    x = observations[4, False][:20]
    rows = x.shape[1]
    rc, rec, status = P.pack(x, 4, False, pitch=2 * rows * 34, n=10)
    assert rc == 0 and not status.any()
    rc, y = P.unpack(rec, np.arange(10), 4, False)
    assert np.array_equal(_bits(y), _bits(x[::2]))


def test_argument_checks_and_bad_indices(observations):
    x = observations[1, False][:4]
    assert P.pack(x, 0, False)[0] == -2 and P.pack(x, 1, 2)[0] == -2
    assert P.pack(x, 1, False, pitch=938 * 34 - 1)[0] == -2
    rc, rec, _ = P.pack(x, 1, False)
    assert P.unpack(rec, [0], 5, False)[0] == -2
    rc, y = P.unpack(rec, [-1, 4, 1 << 40, 2], 1, False)  # outside [0, n_records): an all-zero observation
    assert rc == 0 and not y[:3].any() and np.array_equal(_bits(y[3]), _bits(x[2]))
