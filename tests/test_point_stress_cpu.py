"""The CPU twin of tests/test_gpu_point_stress.py: the generators' self-checks, and the small cases of the variable-base point
kernels (lag_scalar_mul, k_scale_powers, k_lag_stage, k_lag_finish) through the kernel emulation of tests/emu, compared limb for
limb with the oracle's C port and the big-int restatement of ToLagrangeG1 (generators and references in tests/point_stress.py).

The emulation libraries are the ones of tests/test_emu_mpcsetup_cpu.py and tests/test_emu_lagrange_cpu.py.  Their calls run in a
pool of spawned worker processes, one call per job, so that the thirteen groups share the host's cores."""
import multiprocessing
import os
import random
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import pytest

from tests import lagrange_ref as LR
from tests import point_stress as S
from tests.test_emu_lagrange_cpu import _lib as _lagrange_lib
from tests.test_emu_lagrange_cpu import emu_to_lagrange
from tests.test_emu_mpcsetup_cpu import _lib as _mpc_lib
from tests.test_emu_mpcsetup_cpu import emu_scale_powers


@pytest.fixture(scope="module")
def pool():
    """map over spawned worker processes (the emulation keeps its thread indices in globals: one call per process at a time)"""
    _mpc_lib()   # built once, here, before the workers load it
    _lagrange_lib()
    ex = ProcessPoolExecutor(max_workers=max(1, os.cpu_count() or 1), mp_context=multiprocessing.get_context("spawn"))
    try:
        yield lambda f, jobs: list(ex.map(f, jobs))
    finally:
        ex.shutdown(cancel_futures=True)


# ---- the generators ----
@pytest.mark.parametrize("name", S.GROUPS)
def test_digit_cases_round_trip(name):
    """every planned digit vector of family A comes back from the restated DigitStream, every scalar recomposes, and r - 2 takes
    xyzz_add's doubling branch at the ladder's last addition for W = 3 ... 6 (the one exception: secp256k1 at W = 7, whose r is
    not 1 mod 2^7)"""
    q = S.group(name).fr.q
    for W in S.WIDTHS:
        nw = S.nwin(name, W)
        cases = S.digit_cases(name, W)
        names = [c for c, _, _ in cases]
        assert len(set(names)) == len(names) and {"all-min", "all-max", "r-2", "2^W-1"} <= set(names)
        assert "alt-min-max" in names or "alt-max-min" in names, (name, W)
        # every window; at the highest one below the top, a negative digit needs a top digit 1 that may not fit below r
        assert sum(c.startswith("single") for c in names) >= 3 * (nw - 1) - 2, (name, W)
        assert any(c.startswith("top max") for c in names), (name, W)
        for case, s, ds in cases:
            got = S.digit_stream(s, W, nw)
            assert 0 < s < q and S.compose(got, W) == s, (name, W, case, s)
            assert ds is None or got == ds, (name, W, case, s, got, ds)
            assert all(-(1 << (W - 1)) <= d < (1 << (W - 1)) for d in got[:-1]) and 0 <= got[-1] <= 1 << (W - 1), (name, W, case)
    for W in (3, 4, 5, 6, 7):
        adds = S.ladder_additions(q - 2, W, S.nwin(name, W), q)
        doubling = adds[-1] == (0, "double")
        assert doubling == (q % (1 << W) == 1), (name, W, adds[-1])
        assert doubling or (name, W) == ("secp256k1_g1", 7)
        assert all(b == "add" for _, b in adds[:-1]), (name, W)
    # no other family-A scalar reaches the doubling or the cancellation branch
    for W in S.WIDTHS:
        for case, s, _ in S.digit_cases(name, W):
            if case != "r-2":
                assert all(b == "add" for _, b in S.ladder_additions(s, W, S.nwin(name, W), q)), (name, W, case)


@pytest.mark.parametrize("curve", LR.CURVES)
def test_planted_stages_and_ramp(curve):
    """family C's plan covers every case at j = 0, 1 and h - 1 of every stage in separate butterflies, and its input logs give the
    planted relations when the stages are run forward (planted_logs asserts it); the ramp's closed form equals the scalar-domain
    restatement at n = 16"""
    for n in (16, 32, 1024):
        trs = S.planted_transforms(curve, n, 7)
        for s in range(n.bit_length() - 1):
            plans = [p for t, p, _ in trs if t == s]
            flat = [(c, j) for p in plans for c, _, j in p]
            assert sorted(flat) == sorted((c, j) for c in S.PLANT_CASES for j in S.plant_positions(n, s))
            for p in plans:
                assert len({(b, j) for _, b, j in p}) == len(p)
    n = 16
    assert S.ramp_lagrange(curve, n, range(n)) == LR.to_lagrange_scalars(curve, list(range(1, n + 1)))
    idx = S.sample_indices(1 << 20, 1)
    assert len(idx) == 4096 and {0, 1, (1 << 19) - 1, 1 << 19, (1 << 19) + 1, (1 << 20) - 2, (1 << 20) - 1} <= set(idx)


def test_mask_layout():
    inf = S.mask_layout()
    masks = {sum(inf[S.SCALE_M * t + b] << b for b in range(S.SCALE_M)) for t in range(S.MASK_THREADS)}
    assert masks == set(range(256)) and not any(inf[S.MASK_THREADS * S.SCALE_M :])


# ---- A: the ladder (k_scale_powers) ----
def _scale_job(job):
    name, family, case, pts, c, r, start = job
    q = S.group(name).fr.q
    got = emu_scale_powers(name, pts, c, r, start)
    ss = S.geometric_scalars(q, c * pow(r, start, q), r, pts.shape[0])
    S.compare("%s A %s %s" % (name, family, case), got, S.expected_scaled((name, pts, ss)), ss)


def test_ladder_scalars_emulated(pool):
    """family A on the CPU, all thirteen groups: the named digit cases (r - 1, r - 2, r - 3, (r +- 1)/2, 2^(W-1), 2^(W-1) + 1,
    2^W - 1) and the all-minimum / all-maximum digit vectors as c with r = 1, and the geometric families (r - 2, 1) and
    (r - 2, r - 1), on 19 points (two full threads and a tail of 3) with one infinity that moves from call to call.  (r - 2) is the
    doubling branch of the ladder's last addition."""
    jobs = []
    for name in S.GROUPS:
        ks, pts = S.random_points(name, S.CALL_POINTS, 11)
        q = S.group(name).fr.q
        W = S.scale_w(name)
        calls = [("digits", case, s, 1) for case, s, ds in S.digit_cases(name, W) if ds is None or case in ("all-min", "all-max")]
        calls += [("geometric", fam, *S.geometric(name, fam)[:2]) for fam in ("-2,1", "-2,-1")]
        for k, (family, case, c, r) in enumerate(calls):
            p, _ = S.with_infinity(pts, ks, k % S.CALL_POINTS)
            jobs.append((name, family, "%s W=%d" % (case, W), p, c, r, 0))
        assert len(calls) == 12 and q > 2
    pool(_scale_job, jobs)


# ---- B: the infinity masks of the shared inversion (k_scale_powers) ----
def test_mask_normalisation_emulated(pool):
    """family B on the CPU, all thirteen groups: 256 threads carrying every infinity mask, then a tail of 5, out[i] =
    [3 (-1)^i] [i + 1]G.  The call is cut into sub-calls of 32 whole threads continuing the powers (start), so the groups share
    the workers; each thread sees what it sees in one call."""
    jobs = []
    for name in S.GROUPS:
        q = S.group(name).fr.q
        ks_in, _ = S.mask_logs(name, 3, q - 1)
        pts = S.expected_multiples((name, ks_in))
        step = 32 * S.SCALE_M
        for lo in range(0, S.MASK_N, step):
            jobs.append((name, "B", "masks from thread %d" % (lo // S.SCALE_M), pts[lo : lo + step], 3, q - 1, lo))
    pool(_scale_job, jobs)


# ---- C: planted collisions at every stage of ToLagrangeG1 ----
def _lagrange_job(job):
    curve, n, s, plan, logs = job
    pts = S.expected_multiples((curve + "_g1", logs))
    got = emu_to_lagrange(curve, pts)
    if n <= 16:
        want = S.lagrange_points_ref((curve, logs))
    else:
        want = S.expected_multiples((curve + "_g1", LR.to_lagrange_scalars(curve, logs)))
    S.compare("%s C n=%d stage %d: %s" % (curve, n, s, S.plan_text(plan)), got, want)


def test_planted_stages_emulated(pool):
    """family C on the CPU, seven curves: n = 16 against the point-domain restatement, n = 32 against the scalar-domain one"""
    jobs = [(c, n, s, plan, logs) for c in LR.CURVES for n in (16, 32) for s, plan, logs in S.planted_transforms(c, n, 3 + n)]
    random.Random(0).shuffle(jobs)
    pool(_lagrange_job, jobs)
