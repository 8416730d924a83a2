"""The grid front end's cell-ordered points and block table (sgb_grid.cu) against an exact model.

Every coordinate here is a small multiple of 1/64 and both boxes are centred on the origin, so the device's FP32 centred coordinates,
differences and squared distances are all exact: a numpy brute force in FP64 IS the FP32 search, ties included.  Two corner points at
+-1000 m stretch the box to 2000 m, which pins the cell to 2000 / 8000 = 0.25 m (the cell-count bound) with the origin at -1000 m, so
every lattice line at a multiple of 0.25 m lies exactly on a cell face.
"""
import re

import numpy as np
import pytest

import np_factors as NF

pytestmark = pytest.mark.gpu

H = 1.0 / 16  # lattice spacing
CELL = 0.25
CORNERS = np.array([[-1000.0, -1000.0, -1000.0], [1000.0, 1000.0, 1000.0]])


def _target(extra=None):
    g = np.arange(64) * H
    floor = np.array([[x, y, 0.0] for x in g for y in g])  # z = 0, x and y in [0, 4)
    wall = np.array([[2.0 + H / 2, y, z] for y in g for z in g[1:32]])  # x = 2.03125
    dup = np.repeat(floor[:300:3], 3, axis=0)  # 100 points with three more copies each, at other leaf positions
    parts = [floor, wall, dup] + ([extra] if extra is not None else []) + [CORNERS]
    return np.concatenate(parts)


def _source(rng, extra=None):
    g = np.arange(64) * H
    base = np.array([[x, y, 0.0] for x in g[::2] for y in g[::2]])
    near = base + rng.integers(-3, 4, base.shape) / 64.0  # settled by the probe
    centres = np.array([[x + CELL / 2, y + CELL / 2, 0.0] for x in np.arange(16) * CELL for y in np.arange(16) * CELL])  # u - 1/2 integral
    faces = np.array([[x, y, z] for x in np.arange(16) * CELL for y in np.arange(16) * CELL for z in (0.0, CELL)])  # on cell faces
    high = base[::7] + np.array([0.0, 0.0, 1.0]) * (rng.integers(10, 32, (len(base[::7]), 1)) / 64.0)  # nothing within half a cell: ring
    parts = [near, centres, faces, high] + ([extra] if extra is not None else []) + [CORNERS]
    return np.concatenate(parts)


def _brute(tgt, q):
    d = np.empty((len(q), len(tgt)))
    for a in range(0, len(q), 256):
        d[a : a + 256] = ((q[a : a + 256, None, :] - tgt[None, :, :]) ** 2).sum(-1)
    return d.min(1), d


def _grid_line(err):
    m = re.findall(r"\[sgb\] grid front end: cell \S+ \(origin (\S+) (\S+) (\S+), inv_cell (\S+)\), (\d+) key bits, (\d+) blocks, largest block (\d+) points, "
                   r"[\d.]+ B/point(, dropped)?", err)
    assert len(m) == 1, err
    o = [float.fromhex(x) for x in m[0][:3]]
    return o, float.fromhex(m[0][3]), int(m[0][6]), bool(m[0][7])


def _run(tgt, src, profiling):
    import small_gicp_b200 as sg

    ctx = sg.Context(0, profiling=profiling)
    ctx.set_target(tgt)
    ctx.build_target_kdtree(0)
    ctx.set_source(src)
    ctx.linearize(np.eye(4), factor=sg.FACTOR_ICP, rejector=sg.REJECT_DISTANCE, max_dist_sq=1.0)
    corr = ctx.correspondences()
    ctx.close()
    return corr


def _check_exact(tgt, src, corr):
    dmin, d = _brute(tgt, src)
    assert np.all(corr != NF.NO)
    got = d[np.arange(len(src)), corr.astype(np.int64)]
    assert np.array_equal(got, dmin), np.nonzero(got != dmin)[0][:10]
    # exact duplicates (same coordinates, different leaf positions): the device picks the lowest leaf position among them.  Leaf
    # positions are not visible from here, so what is checked is the consequence: every query whose tied nearest points are copies of
    # ONE point gets the same copy, whichever path (probe, ring, tree walk) answered it
    chosen = {}
    for i in range(len(src)):
        ties = np.nonzero(d[i] == dmin[i])[0]
        if len(ties) > 1 and np.all(tgt[ties] == tgt[ties[0]]):
            key = tuple(tgt[ties[0]])
            assert chosen.setdefault(key, int(corr[i])) == int(corr[i]), (i, key)
    return len(chosen)


def _pending(err):
    m = re.findall(r"\[sgb\] grid front end: (\d+) of (\d+) queries pending", err)
    assert len(m) == 1, err
    return int(m[0][0])


def test_probe_exact_against_fp32_brute_force(capfd, monkeypatch):
    """probe + ring over the block table: bit-exact nearest distances, duplicates resolved consistently, points and queries on cell
    faces and at cell centres.  The profiling build finishes EVERY pending query warp-per-query (ring phase, SGB_PENDING_DIV=1); the
    product library, with more pending queries than its split, finishes them with the packet walk -- both must give the same answer."""
    rng = np.random.default_rng(5)
    tgt, src = _target(), _source(rng)
    monkeypatch.setenv("SGB_DEBUG_PENDING", "1")
    monkeypatch.setenv("SGB_PENDING_DIV", "1")
    capfd.readouterr()
    corr_prof = _run(tgt, src, profiling=True)
    err = capfd.readouterr().err
    origin, inv_cell, largest, dropped = _grid_line(err)
    assert origin == [-1000.0] * 3 and inv_cell == 1.0 / CELL, (origin, inv_cell)  # the exact model's premise: faces at multiples of 0.25
    assert not dropped and 64 <= largest < 2048
    # the probe settles exactly the queries whose nearest point lies within the settle radius ((1/2 - 4e-3) cells, FP32); the rest
    # (the raised queries, ~20 %) went through the ring phase
    settle_d2 = np.float32(((0.5 - 4e-3) * CELL) ** 2)
    dmin, _ = _brute(tgt, src)
    want_pending = int((dmin > settle_d2).sum())
    assert want_pending > 200 and _pending(err) == want_pending, (_pending(err), want_pending)
    monkeypatch.delenv("SGB_DEBUG_PENDING")
    monkeypatch.delenv("SGB_PENDING_DIV")
    corr = _run(tgt, src, profiling=False)
    assert np.array_equal(corr, corr_prof)
    assert _check_exact(tgt, src, corr) > 10  # queries that met a duplicated point


@pytest.mark.parametrize("k", [2048, 2049])
def test_largest_block_limit(k, capfd, monkeypatch):
    """a block of exactly kGridMaxList points keeps the front end, one more point drops it (the tree search alone answers); the block
    size is the sum of its four runs.  Exact either way."""
    rng = np.random.default_rng(6)
    spot = np.array([500.0 + H, 500.0 + H, 500.0 + H])  # k copies of one point, far from everything else: one block of exactly k points
    tgt = _target(np.repeat(spot[None], k, axis=0))
    src = _source(rng, spot[None] + np.array([[0.0, 0.0, 0.0], [1 / 64, 0.0, 0.0], [0.0, -1 / 32, 1 / 64]]))
    monkeypatch.setenv("SGB_DEBUG_PENDING", "1")
    capfd.readouterr()
    corr = _run(tgt, src, profiling=True)
    err = capfd.readouterr().err
    _, inv_cell, largest, dropped = _grid_line(err)
    assert inv_cell == 1.0 / CELL and largest == k
    assert dropped == (k > 2048)
    assert ("queries pending" in err) == (k <= 2048)
    dmin, d = _brute(tgt, src)
    got = d[np.arange(len(src)), corr.astype(np.int64)]
    assert np.array_equal(got, dmin)
