"""Host-side mirror of the reference interface for the MultiExp path, over the C ABI.

Reference (Go): `func (p *G1Jac) MultiExp(points []G1Affine, scalars []fr.Element,
config ecc.MultiExpConfig) (*G1Jac, error)` -- ecc/bn254/multiexp.go:32 (G1Affine :20, G2Jac :357,
G2Affine :345; ecc/bls12-381/multiexp.go:20,32,343,355); `ecc.MultiExpConfig{NbTasks int}` --
ecc/ecc.go:107-110.  Same names, argument meaning and error behaviour:
  * len(points) != len(scalars)  -> error "len(points) != len(scalars)"   (multiexp.go:61-64)
  * config.NbTasks > 1024        -> error "invalid config: config.NbTasks > 1024"  (:69-71)
  * the receiver is overwritten and returned.

Points and scalars are numpy uint64 arrays holding exactly the bytes Go holds (Montgomery limbs,
little-endian; infinity = all-zero point); see include/gmsm.h.  There is no Go toolchain in this
environment, so this Python mirror (ctypes) is the host side the parity tests drive; the cgo shim a
maintainer would add is in INTEGRATION.md.
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass

import numpy as np

from . import _native
from .curves import CURVES, GROUPS


class MultiExpError(Exception):
    """the Go `error` value"""


@dataclass
class MultiExpConfig:
    """ecc.MultiExpConfig (ecc/ecc.go:107-110)"""

    NbTasks: int = 0


def _check(rc):
    if rc != 0:
        raise MultiExpError(_native.last_error())


def _handle(h):
    """a handle the library returned; NULL is its error"""
    if not h:
        raise MultiExpError(_native.last_error())
    return h


def _as_u64(a, cols, what):
    a = np.ascontiguousarray(a, dtype=np.uint64)
    if a.ndim == 1:
        if a.size % cols:
            raise ValueError("%s: size %d is not a multiple of %d u64 words" % (what, a.size, cols))
        a = a.reshape(-1, cols)
    if a.ndim != 2 or a.shape[1] != cols:
        raise ValueError("%s: expected shape (n, %d) uint64, got %r" % (what, cols, a.shape))
    return a


class _Point:
    GROUP = None  # set by curve_package()
    WORDS = 0

    def __init__(self, limbs=None):
        self.limbs = np.zeros(self.WORDS, dtype=np.uint64) if limbs is None else np.array(limbs, dtype=np.uint64).reshape(self.WORDS)

    def __eq__(self, o):
        return type(self) is type(o) and np.array_equal(self.limbs, o.limbs)

    def __repr__(self):
        return "%s(%s)" % (type(self).__name__, " ".join("%016x" % int(v) for v in self.limbs))


class _JacBase(_Point):
    def MultiExp(self, points, scalars, config: MultiExpConfig = None):
        """(*G1Jac).MultiExp / (*G2Jac).MultiExp -- one-shot, host buffers (gmsm_multiexp)."""
        config = config or MultiExpConfig()
        g = self.GROUP
        w = g.words
        points = _as_u64(points, 2 * w, "points")
        scalars = _as_u64(scalars, g.scalar_words, "scalars")
        if points.shape[0] != scalars.shape[0]:
            raise MultiExpError("len(points) != len(scalars)")  # multiexp.go:61-64
        out = np.zeros(3 * w, dtype=np.uint64)
        L = _native.lib()
        rc = L.gmsm_multiexp(g.id, points.ctypes.data, scalars.ctypes.data, points.shape[0], int(config.NbTasks), out.ctypes.data)
        _check(rc)
        self.limbs = out
        return self

    # coordinates as u64 limb arrays
    @property
    def X(self):
        return self.limbs[: self.WORDS // 3]

    @property
    def Y(self):
        return self.limbs[self.WORDS // 3 : 2 * self.WORDS // 3]

    @property
    def Z(self):
        return self.limbs[2 * self.WORDS // 3 :]

    def IsInfinity(self):
        return not self.Z.any()


class _AffBase(_Point):
    JAC = None

    def MultiExp(self, points, scalars, config: MultiExpConfig = None):
        """(*G1Affine).MultiExp (multiexp.go:20-27): Jacobian MultiExp then FromJacobian."""
        j = self.JAC()
        j.MultiExp(points, scalars, config)
        return self.FromJacobian(j)

    def FromJacobian(self, j):
        """g1.go:150-166.  The engine returns the affine-normalised representative (X, Y, One) or
        (0,0,0), so FromJacobian is a copy of X, Y (Z^-1 = One)."""
        w = self.WORDS // 2
        self.limbs = np.concatenate([j.limbs[:w], j.limbs[w : 2 * w]]) if j.Z.any() else np.zeros(self.WORDS, dtype=np.uint64)
        return self

    @property
    def X(self):
        return self.limbs[: self.WORDS // 2]

    @property
    def Y(self):
        return self.limbs[self.WORDS // 2 :]

    def IsInfinity(self):
        return not self.limbs.any()


def curve_package(curve: str):
    """Returns (G1Affine, G1Jac, G2Affine, G2Jac) bound to `curve` in {"bn254", "bls12381", "bls12377", "secp256k1", "bw6761", "bls24315", "bls24317", "bw6633"}
    -- the analogue of importing ecc/bn254, ecc/bls12-381, ... (no G2 for secp256k1; none provided for bls24-315 / bls24-317: None, None)."""
    out = []
    for grp in ("g1", "g2"):
        if "%s_%s" % (curve, grp) not in CURVES:   # secp256k1: G1 only
            out += [None, None]
            continue
        g = GROUPS["%s_%s" % (curve, grp)]
        jac = type("%s_%sJac" % (curve, grp.upper()), (_JacBase,), {"GROUP": g, "WORDS": 3 * g.words})
        aff = type("%s_%sAffine" % (curve, grp.upper()), (_AffBase,), {"GROUP": g, "WORDS": 2 * g.words, "JAC": jac})
        out += [aff, jac]
    return tuple(out)


# default names = the bn254 package (BASELINE.json's headline curve)
G1Affine, G1Jac, G2Affine, G2Jac = curve_package("bn254")


class ResidentBases:
    """gmsm_bases_*: bases uploaded once (SRS / proving key), scalars per call from host memory."""

    def __init__(self, curve: str, points, device: int = 0):
        self.cid = CURVES[curve]
        self.w = GROUPS[curve].words
        self.sw = GROUPS[curve].scalar_words
        points = _as_u64(points, 2 * self.w, "points")
        self.n = points.shape[0]
        self._h = _handle(_native.lib().gmsm_bases_upload(self.cid, points.ctypes.data, self.n, device))

    def MultiExp(self, scalars, config: MultiExpConfig = None, offset: int = 0):
        config = config or MultiExpConfig()
        scalars = _as_u64(scalars, self.sw, "scalars")
        out = np.zeros(3 * self.w, dtype=np.uint64)
        rc = _native.lib().gmsm_bases_multiexp(self._h, offset, scalars.ctypes.data, scalars.shape[0], int(config.NbTasks), out.ctypes.data)
        _check(rc)
        return out

    def MultiExpDevice(self, d_scalars, n: int = None, config: MultiExpConfig = None, offset: int = 0, stream=None):
        """the same with scalars already on the device (torch int64 tensor in fr.Element layout, e.g. straight out of
        fft.Domain.fft_device): nothing but the 96..288-byte result crosses PCIe"""
        config = config or MultiExpConfig()
        if n is None:
            n = d_scalars.numel() // self.sw
        out = np.zeros(3 * self.w, dtype=np.uint64)
        rc = _native.lib().gmsm_bases_multiexp_device(self._h, offset, d_scalars.data_ptr(), n, int(config.NbTasks), out.ctypes.data, stream)
        _check(rc)
        return out

    def Precompute(self, c: int = 0) -> int:
        """gmsm_bases_precompute: replace the device copy of the bases by window tables (row j = 2^(c*j) * bases);
        later MultiExp calls are bit-identical and faster.  Returns the table window width."""
        _check(_native.lib().gmsm_bases_precompute(self._h, int(c)))
        return _native.lib().gmsm_bases_table_bits(self._h)

    def close(self):
        if self._h:
            _native.lib().gmsm_bases_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Engine:
    """Device-level engine (gmsm_ctx_*): inputs already resident in HBM as torch uint8/int64 tensors.
    torch is used for device memory and streams only."""

    def __init__(self, curve: str, max_n: int, c: int = 0, device: int = 0, tables: bool = False):
        import torch

        self.torch = torch
        self.curve = curve
        self.cid = CURVES[curve]
        self.w = GROUPS[curve].words
        self.sw = GROUPS[curve].scalar_words   # u64 words per scalar
        self.device = device
        self.tables = tables
        L = _native.lib()
        self._h = _handle((L.gmsm_ctx_create_tables if tables else L.gmsm_ctx_create)(self.cid, max_n, c, device))
        self.c = L.gmsm_ctx_window_bits(self._h)
        self.nwin = L.gmsm_ctx_num_windows(self._h)
        self.workspace_bytes = L.gmsm_ctx_workspace_bytes(self._h)
        self.partials_bytes = self.nwin * 4 * self.w * 8
        dev = torch.device("cuda", device)
        self._out = torch.zeros(3 * self.w, dtype=torch.int64, device=dev)
        self._partials = torch.zeros(self.partials_bytes // 8, dtype=torch.int64, device=dev)

    # ---- helpers ----
    def _stream(self):
        return ctypes.c_void_p(self.torch.cuda.current_stream(self.device).cuda_stream)

    def to_device(self, arr: np.ndarray):
        t = self.torch.from_numpy(np.ascontiguousarray(arr, dtype=np.uint64).view(np.int64))
        return t.to(self.torch.device("cuda", self.device))

    def msm(self, d_points, d_scalars, n: int = None):
        """full MSM on device tensors; returns the device tensor holding the Jacobian triple (int64 view)."""
        if n is None:
            n = d_scalars.numel() // self.sw
        rc = _native.lib().gmsm_ctx_msm_device(self._h, d_points.data_ptr(), d_scalars.data_ptr(), n, self._out.data_ptr(), self._stream())
        _check(rc)
        return self._out

    # ---- window-table mode (Engine(..., tables=True)) ----
    def build_tables(self, d_points, n: int = None):
        """device tensor of nwin rows of n affine points, row j = 2^(c*j) * points (gmsm_tables_build_device)"""
        if n is None:
            n = d_points.numel() // (2 * self.w)
        tab = self.torch.empty(self.nwin * n * 2 * self.w, dtype=self.torch.int64, device=d_points.device)
        with self.torch.cuda.device(self.device):
            rc = _native.lib().gmsm_tables_build_device(self.cid, self.c, d_points.data_ptr(), n, tab.data_ptr(), n, self._stream())
        _check(rc)
        return tab

    def msm_tables(self, d_table, row_stride: int, d_scalars, n: int = None, offset: int = 0):
        if n is None:
            n = d_scalars.numel() // self.sw
        rc = _native.lib().gmsm_ctx_msm_tables_device(self._h, d_table.data_ptr(), row_stride, offset, d_scalars.data_ptr(), n,
                                                      self._out.data_ptr(), self._stream())
        _check(rc)
        return self._out

    def msm_host_result(self, d_points, d_scalars, n: int = None) -> np.ndarray:
        return self.msm(d_points, d_scalars, n).cpu().numpy().view(np.uint64).copy()

    def window_sums(self, d_points, d_scalars, n: int = None, out=None):
        if n is None:
            n = d_scalars.numel() // self.sw
        out = self._partials if out is None else out
        rc = _native.lib().gmsm_ctx_window_sums_device(self._h, d_points.data_ptr(), d_scalars.data_ptr(), n, out.data_ptr(), self._stream())
        _check(rc)
        return out

    def finalize(self, d_partials, nranks: int):
        rc = _native.lib().gmsm_ctx_finalize_device(self._h, d_partials.data_ptr(), nranks, self._out.data_ptr(), self._stream())
        _check(rc)
        return self._out

    def generate_multiples(self, base_affine: np.ndarray, start: int, n: int):
        """device tensor of n affine points [start + i] * base (SURVEY.md K6)"""
        base_affine = np.ascontiguousarray(base_affine, dtype=np.uint64).reshape(2 * self.w)
        out = self.torch.empty(n * 2 * self.w, dtype=self.torch.int64, device=self.torch.device("cuda", self.device))
        rc = _native.lib().gmsm_generate_multiples_device(self.cid, base_affine.ctypes.data, start, n, out.data_ptr(), self._stream())
        _check(rc)
        return out

    def set_profiling(self, on):
        """True / 1: stage timings (last_stage_ms); 2: also the scatter / accumulate timeline (last_timeline_ms)"""
        _native.lib().gmsm_ctx_set_profiling(self._h, int(on))

    def last_stage_ms(self):
        buf = (ctypes.c_float * 8)()
        rc = _native.lib().gmsm_ctx_last_stage_ms(self._h, buf)
        _check(rc)
        return list(buf)

    def last_timeline_ms(self):
        """the last call's timeline (gmsm_ctx_last_timeline_ms) as a dict: passes = [(stream, start, end)] in pass order,
        stream "main" or "aux"; parts = [(start, end)] of the accumulate parts; ms from the start of the call"""
        L = _native.lib()
        cnt = ctypes.c_int(0)
        buf = (ctypes.c_float * 512)()
        _check(L.gmsm_ctx_last_timeline_ms(self._h, buf, len(buf), ctypes.byref(cnt)))
        v = list(buf)[: cnt.value]
        npass, split, nparts = int(v[0]), int(v[1]), int(v[2])
        ev = v[3:]
        passes = [("main" if r < split else "aux", ev[2 * r], ev[2 * r + 1]) for r in range(npass)]
        parts = [(ev[2 * npass + 2 * k], ev[2 * npass + 2 * k + 1]) for k in range(nparts)]
        return {"passes": passes, "split": split, "parts": parts}

    @property
    def last_launches(self):
        return _native.lib().gmsm_ctx_last_launches(self._h)

    def close(self):
        if self._h:
            _native.lib().gmsm_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def BatchScalarMultiplication(curve: str, base, scalars) -> np.ndarray:
    """BatchScalarMultiplicationG1 / G2 (ecc/bn254/g1.go:1039-1118, g2.go:1001+): multiplies the same
    base by all scalars; returns the points in affine coordinates, shape (n, 2*words) uint64."""
    g = GROUPS[curve]
    base = np.ascontiguousarray(base, dtype=np.uint64).reshape(2 * g.words)
    scalars = _as_u64(scalars, g.scalar_words, "scalars")
    out = np.zeros((scalars.shape[0], 2 * g.words), dtype=np.uint64)
    rc = _native.lib().gmsm_batch_scalar_mul(g.id, base.ctypes.data, scalars.ctypes.data, scalars.shape[0], out.ctypes.data)
    _check(rc)
    return out


# ---- test hooks ----
def test_op(curve: str, op: int, a: np.ndarray, b: np.ndarray, out_words: int) -> np.ndarray:
    a = np.ascontiguousarray(a, dtype=np.uint32)
    n = a.shape[0]
    b = np.ascontiguousarray(b, dtype=np.uint32) if b is not None else np.zeros((n, 1), dtype=np.uint32)
    out = np.zeros((n, out_words), dtype=np.uint32)
    rc = _native.lib().gmsm_test_op(CURVES[curve], op, a.ctypes.data, b.ctypes.data, out.ctypes.data, n)
    _check(rc)
    return out


def test_digits(curve: str, c: int, scalars: np.ndarray) -> np.ndarray:
    g = GROUPS[curve]
    scalars = _as_u64(scalars, g.scalar_words, "scalars")
    n = scalars.shape[0]
    W = (g.scalar_bits + c - 1) // c
    out = np.zeros((W, n), dtype=np.uint32)
    rc = _native.lib().gmsm_test_digits(g.id, c, scalars.ctypes.data, n, out.ctypes.data)
    _check(rc)
    return out
