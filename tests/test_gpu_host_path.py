"""Host-facing behaviour of the C ABI on a GPU box (SURVEY.md section 8b: ownership / lifetime / threading of the drop-in
boundary): pageable caller buffers through the pinned staging ring, error paths that leave no work in flight, concurrent
calls (the reference is called from several goroutines at once, multiexp_test.go:385-415), the lane-parallel tail kernels
and the serialisation of device-level calls that share one context."""
import ctypes
import threading

import numpy as np
import pytest

from oracle import cref
from tests.gpu_common import make_inputs

pytestmark = pytest.mark.gpu


def _pkg():
    import gnark_crypto_b200 as pkg

    return pkg


def _native():
    import importlib

    return importlib.import_module("gnark-crypto_b200._native")


def _oneshot(g, pts, s):
    pkg = _pkg()
    cid = pkg.CURVES[g]
    out = np.zeros(pts.shape[1] // 2 * 3, dtype=np.uint64)
    rc = _native().lib().gmsm_multiexp(cid, pts.ctypes.data, s.ctypes.data, pts.shape[0], 0, out.ctypes.data)
    return rc, out


@pytest.mark.parametrize("g,n", [("bn254_g1", (1 << 19) + 12345), ("bls12381_g1", 300001), ("bn254_g2", 150000)])
def test_pageable_and_pinned_host_buffers_agree(g, n, monkeypatch):
    """the same call on pageable numpy arrays (staged through the library's pinned ring, several 8 MiB slots and batches),
    on pinned memory (direct asynchronous copies) and with the ring disabled must give the oracle's result"""
    import torch

    pts, s = make_inputs(g, n, 99)
    want, _, _, _ = cref.msm(g, pts, s, c=0, nthreads=8)
    w = pts.shape[1]
    rc, out = _oneshot(g, pts, s)
    assert rc == 0 and np.array_equal(out[:w], want)
    hp = torch.from_numpy(pts.view(np.int64).reshape(-1).copy()).pin_memory()
    hs = torch.from_numpy(s.view(np.int64).reshape(-1).copy()).pin_memory()
    rc, out2 = _oneshot(g, hp.numpy().view(np.uint64).reshape(n, w), hs.numpy().view(np.uint64).reshape(n, 4))
    assert rc == 0 and np.array_equal(out2, out)
    monkeypatch.setenv("GMSM_STAGING", "0")
    rc, out3 = _oneshot(g, pts, s)
    assert rc == 0 and np.array_equal(out3, out)
    monkeypatch.setenv("GMSM_STAGING", "1")
    monkeypatch.setenv("GMSM_COPY_THREADS", "1")   # (read once per process: only documents the knob)
    rc, out4 = _oneshot(g, pts, s)
    assert rc == 0 and np.array_equal(out4, out)


def test_fault_mid_pipeline_leaves_nothing_in_flight(monkeypatch):
    """force an error after the first batches were enqueued (copies and kernels then busy on three streams): the call must
    return the error with every stream drained -- the host buffers are overwritten right away and the next calls, which
    reuse the session's device buffers, must still be exact (run under compute-sanitizer by tools/gpu_sanitize.sh)"""
    g = "bn254_g1"
    n = (1 << 21) + 77     # five geometric batches
    pts, s = make_inputs(g, n, 5)
    want, _, _, _ = cref.msm(g, pts, s, c=0, nthreads=8)
    for k in (0, 2):
        p2, s2 = pts.copy(), s.copy()
        monkeypatch.setenv("GMSM_FAULT_AFTER_BATCH", str(k))
        rc, _ = _oneshot(g, p2, s2)
        assert rc != 0 and "injected fault" in _native().last_error()
        p2[:] = 0xFFFFFFFFFFFFFFFF       # reuse of the caller's memory the moment the call returned
        s2[:] = 0
        monkeypatch.delenv("GMSM_FAULT_AFTER_BATCH")
        rc, out = _oneshot(g, pts, s)
        assert rc == 0 and np.array_equal(out[: pts.shape[1]], want)


def test_concurrent_calls_from_several_threads():
    """BenchmarkManyMultiExpG1Reference (multiexp_test.go:385-415): several goroutines, each one MultiExp.  Six host threads,
    two curves, each with its own inputs, twice over; every result bit-exact.  (The session pool holds 3 sessions per
    (curve, device): the fourth concurrent call of a pair waits for a lease.)"""
    jobs = []
    for k, (g, n) in enumerate([("bn254_g1", 200000), ("bn254_g1", 150001), ("bn254_g1", 99999), ("bn254_g1", 70000),
                                ("bls12381_g1", 120000), ("bn254_g2", 60000)]):
        pts, s = make_inputs(g, n, 1000 + k)
        want, _, _, _ = cref.msm(g, pts, s, c=0, nthreads=8)
        jobs.append((g, pts, s, want))
    errs = []

    def run(j):
        g, pts, s, want = jobs[j]
        for _ in range(2):
            rc, out = _oneshot(g, pts, s)
            if rc != 0 or not np.array_equal(out[: pts.shape[1]], want):
                errs.append((j, rc))

    th = [threading.Thread(target=run, args=(j,)) for j in range(len(jobs))]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs, errs


def test_device_level_calls_on_one_context_from_two_streams():
    """two threads drive ONE engine context from two different CUDA streams (ADVICE r01: the shared workspace used to be
    protected only while a call was being enqueued): the calls are chained on the context's completion event, so both
    results are exact"""
    import torch

    pkg = _pkg()
    g = "bn254_g1"
    n = 150000
    pts, s = make_inputs(g, n, 31)
    pts2, s2 = make_inputs(g, n, 32, start=7)
    want1, _, _, _ = cref.msm(g, pts, s, c=0, nthreads=8)
    want2, _, _, _ = cref.msm(g, pts2, s2, c=0, nthreads=8)
    eng = pkg.Engine(g, n)
    L = _native().lib()
    dev = torch.device("cuda", 0)
    d = [(eng.to_device(pts), eng.to_device(s), torch.zeros(12, dtype=torch.int64, device=dev)),
         (eng.to_device(pts2), eng.to_device(s2), torch.zeros(12, dtype=torch.int64, device=dev))]
    streams = [torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev)]
    torch.cuda.synchronize()
    errs = []

    def run(k):
        dp, ds, do = d[k]
        for _ in range(6):
            rc = L.gmsm_ctx_msm_device(eng._h, dp.data_ptr(), ds.data_ptr(), n, do.data_ptr(), ctypes.c_void_p(streams[k].cuda_stream))
            if rc != 0:
                errs.append(rc)

    th = [threading.Thread(target=run, args=(k,)) for k in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    torch.cuda.synchronize()
    assert not errs
    assert np.array_equal(d[0][2].cpu().numpy().view(np.uint64)[:8], want1)
    assert np.array_equal(d[1][2].cpu().numpy().view(np.uint64)[:8], want2)
    eng.close()


@pytest.mark.parametrize("g,n", [("bn254_g1", 50000), ("bls12381_g1", 20000), ("bn254_g2", 12000), ("bls12381_g2", 6000),
                                 ("bls12377_g1", 20000), ("bls12377_g2", 6000), ("secp256k1_g1", 50000), ("bw6761_g1", 4000),
                                 ("bw6761_g2", 4000), ("bls24315_g1", 30000), ("bls24317_g1", 30000), ("bw6633_g1", 5000),
                                 ("bw6633_g2", 5000)])
@pytest.mark.parametrize("quad", ["0", "1"])
def test_tail_kernels_serial_and_lane_parallel(g, n, quad, monkeypatch):
    """the carry join / bucket reduction / group sums in their one-thread-per-chain and one-quad-per-chain forms (csrc/quad.cuh)
    are both exact, at several widths, with the cross-test ingredients and with every scalar equal (one bucket per window
    spans all the chunks: the carry levels do the work).  All thirteen groups; GMSM_QUAD=0 is the serial form also for the
    bw6 groups, whose default is lane-parallel"""
    monkeypatch.setenv("GMSM_QUAD", quad)
    pkg = _pkg()
    pts, s = make_inputs(g, n, 17)
    want, _, _, _ = cref.msm(g, pts, s, c=0, nthreads=8)
    s_eq = s.copy()
    s_eq[:] = s[3]
    want_eq, _, _, _ = cref.msm(g, pts, s_eq, c=0, nthreads=8)
    w = pts.shape[1]
    for c in (7, 12, 15):
        eng = pkg.Engine(g, n, c=c)
        try:
            dp = eng.to_device(pts)
            assert np.array_equal(eng.msm_host_result(dp, eng.to_device(s), n)[:w], want), c
            assert np.array_equal(eng.msm_host_result(dp, eng.to_device(s_eq), n)[:w], want_eq), c
        finally:
            eng.close()
