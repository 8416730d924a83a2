"""Graduated non-convexity (sgb_align_batch_gnc) without a GPU: the numpy formulas and schedules of tests/np_gnc.py against their
definitions and limits, and the device's own gnc_weight / gnc_stage_begin (sgb_math.cuh, compiled for the host in tests/host_gnc without
FMA contraction) against them bit for bit."""
import ctypes
import math
import os
import subprocess

import numpy as np
import pytest

import np_gnc as G
from conftest import ROOT

HG_DIR = os.path.join(ROOT, "tests", "host_gnc")
c_dp = ctypes.POINTER(ctypes.c_double)


@pytest.fixture(scope="module")
def hg():
    subprocess.check_call(["make", "-s", "-C", HG_DIR])
    lib = ctypes.CDLL(os.path.join(HG_DIR, "libsgb_host_gnc.so"))
    lib.sgbg_schedule.restype = ctypes.c_int
    lib.sgbg_schedule.argtypes = [ctypes.c_int, ctypes.c_double, ctypes.c_double, ctypes.c_int, c_dp]
    return lib


def _p(a):
    return a.ctypes.data_as(c_dp)


def _bits_equal(a, b):
    return np.array_equal(np.asarray(a, dtype=np.float64).view(np.uint64), np.asarray(b, dtype=np.float64).view(np.uint64))


def _host_weight(hg, kind, r2, mu, c2):
    r2, mu, c2 = (np.ascontiguousarray(np.broadcast_to(x, np.shape(r2)), dtype=np.float64) for x in (r2, mu, c2))
    out = np.empty(r2.shape)
    hg.sgbg_weight(kind, ctypes.c_size_t(r2.size), _p(r2), _p(mu), _p(c2), _p(out))
    return out


def _random_inputs(rng, n):
    c2 = 10.0 ** rng.uniform(-4, 2, n)
    mu = 10.0 ** rng.uniform(-3, 4, n)
    r2 = c2 * 10.0 ** rng.uniform(-3, 3, n)
    # exactly on the TLS band edges, one ulp either side, and zero residuals
    lo = (mu / (mu + 1.0)) * c2
    hi = ((mu + 1.0) / mu) * c2
    k = n // 8
    r2[:k] = lo[:k]
    r2[k : 2 * k] = np.nextafter(lo[k : 2 * k], np.inf)
    r2[2 * k : 3 * k] = hi[2 * k : 3 * k]
    r2[3 * k : 4 * k] = np.nextafter(hi[3 * k : 4 * k], 0.0)
    r2[4 * k : 4 * k + 16] = 0.0
    return r2, mu, c2


@pytest.mark.parametrize("kind", [G.GM, G.TLS])
def test_host_weight_bitwise(hg, kind):
    r2, mu, c2 = _random_inputs(np.random.default_rng(11 + kind), 40_000)
    assert _bits_equal(_host_weight(hg, kind, r2, mu, c2), G.weight(kind, r2, mu, c2))


@pytest.mark.parametrize("kind", [G.GM, G.TLS])
def test_host_schedule_bitwise(hg, kind):
    rng = np.random.default_rng(21 + kind)
    for _ in range(2000):
        c2 = 10.0 ** rng.uniform(-4, 2)
        r2max = c2 * 10.0 ** rng.uniform(-2, 4)
        if rng.uniform() < 0.05:
            r2max = 0.0
        max_stages = int(rng.integers(1, 80))
        mus = np.zeros(max_stages)
        n = hg.sgbg_schedule(kind, r2max, c2, max_stages, _p(mus))
        ref = G.schedule(kind, r2max, c2, max_stages)
        assert n == len(ref)
        assert _bits_equal(mus[:n], ref)


def test_tls_continuous_at_band_edges():
    rng = np.random.default_rng(3)
    mu = 10.0 ** rng.uniform(-3, 4, 5000)
    c2 = 10.0 ** rng.uniform(-4, 2, 5000)
    lo, hi = (mu / (mu + 1.0)) * c2, ((mu + 1.0) / mu) * c2
    for edge, value in ((lo, 1.0), (hi, 0.0)):
        for side in (1.0 - 1e-12, 1.0 + 1e-12):
            g = G.weight(G.TLS, edge * side, mu, c2)
            assert np.all(np.abs(g - value) < 1e-10 * (1.0 + mu))  # |dg / d ln r2| is about mu / 2 at the edges
    g = G.weight(G.TLS, 0.5 * (lo + hi), mu, c2)  # strictly inside the band: strictly between 0 and 1 where the band is wide enough
    wide = (hi - lo) > 1e-6 * c2
    assert np.all((g[wide] > 0.0) & (g[wide] < 1.0))


def test_tls_monotone():
    mu, c2 = 3.7, 0.25
    r2 = np.linspace(0.0, 2.0 * c2, 20001)
    g = G.weight(G.TLS, r2, mu, c2)
    assert np.all(np.diff(g) <= 0.0) and g[0] == 1.0 and g[-1] == 0.0


def test_gm_stage_count():
    rng = np.random.default_rng(5)
    for _ in range(3000):
        c2 = 10.0 ** rng.uniform(-3, 1)
        r2max = c2 * 10.0 ** rng.uniform(-1, 5)
        mu_0 = 2.0 * r2max / c2
        if mu_0 <= 1.0:
            assert len(G.schedule(G.GM, r2max, c2, 1000)) == 1
            continue
        k = math.log(mu_0) / math.log(G.FACTOR)
        if abs(k - round(k)) < 1e-6:  # an exact power of 1.4: the rounding of the repeated division decides
            continue
        assert len(G.schedule(G.GM, r2max, c2, 1000)) == math.ceil(k) + 1
        assert len(G.schedule(G.GM, r2max, c2, 3)) == min(3, math.ceil(k) + 1)


def test_gm_schedule_decreases_to_one():
    mus = G.schedule(G.GM, 50.0, 0.1, 1000)
    assert mus[0] == 1000.0 and mus[-1] == 1.0 and all(a > b for a, b in zip(mus, mus[1:]))


def test_tls_stops_when_binary():
    rng = np.random.default_rng(9)
    c2 = 0.04
    for _ in range(50):
        r2 = np.concatenate([rng.uniform(0, 0.5 * c2, 300), rng.uniform(3 * c2, 100 * c2, 200), rng.uniform(0.5 * c2, 3 * c2, 20)])
        stages = G.run_fixed(G.TLS, r2, c2, 1000)
        ones = np.ones(r2.shape, dtype=bool)
        assert G.binary(stages[-1][1], ones)
        assert not any(G.binary(g, ones) for _, g in stages[:-1])
        assert all(b[0] == G.FACTOR * a[0] for a, b in zip(stages, stages[1:]))
        # at the end every weight is the true TLS weight: 1 inside the bound, 0 outside (to the band's width at the last mu)
        mu = stages[-1][0]
        assert np.all(stages[-1][1][r2 <= (mu / (mu + 1.0)) * c2] == 1.0)
        assert np.all(stages[-1][1][r2 >= ((mu + 1.0) / mu) * c2] == 0.0)


def test_tls_no_outliers_single_stage():
    r2 = np.array([0.0, 0.01, 0.02])
    stages = G.run_fixed(G.TLS, r2, 0.04, 64)  # 2 r_max^2 = c^2: no outliers
    assert len(stages) == 1 and stages[0][0] == 0.0 and np.all(stages[0][1] == 1.0)
    assert G.mu0(G.TLS, 0.0, 1.0) == (0.0, True)


def test_limits():
    rng = np.random.default_rng(13)
    r2 = 10.0 ** rng.uniform(-4, 2, 1000)
    c2 = 0.3
    # GM: a convex surrogate (mu -> inf) weighs every point 1; at mu = 1 it is the Geman-McClure weight (c^2 / (r^2 + c^2))^2
    assert np.all(np.abs(G.weight(G.GM, r2, 1e12, c2) - 1.0) < 1e-9)
    assert np.allclose(G.weight(G.GM, r2, 1.0, c2), (c2 / (r2 + c2)) ** 2, rtol=1e-15, atol=0)
    # TLS: mu -> 0 weighs every point of r^2 < c^2 / mu ... near 0 except the smallest; mu -> inf is the truncation at c^2
    g = G.weight(G.TLS, r2, 1e12, c2)
    away = np.abs(r2 - c2) > 1e-6 * c2
    assert np.array_equal(g[away], (r2[away] <= c2).astype(float))
    g0 = G.weight(G.TLS, r2, 1e-12, c2)
    assert np.all(g0[r2 > 1e-3 * c2] < 1e-3)
    assert np.all((0.0 <= G.weight(G.TLS, r2, 0.7, c2)) & (G.weight(G.TLS, r2, 0.7, c2) <= 1.0))
