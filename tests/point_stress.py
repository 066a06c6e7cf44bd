"""Scalars, planted inputs, references and checks for the variable-base point kernels shared by kzg.ToLagrangeG1 and mpcsetup
(lagrange_kernels.cuh: the ladder lag_scalar_mul, k_lag_stage, k_lag_finish; mpc_kernels.cuh: k_scale_powers).

Shared by tests/test_gpu_point_stress.py (the sm_90a kernels through mpcsetup.py, kzg.ToLagrangeG1 and the C ABI) and
tests/test_point_stress_cpu.py (the same kernels on the CPU through the emulation of tests/emu).  Not a conftest.

Points are taken from the prime-order subgroup: [k]G for a known discrete logarithm k, so every expected point is [k']G for a
big-int k' and a group-law branch of a kernel is a congruence between discrete logarithms.  `digit_stream` and
`ladder_additions` restate the ladder on those integers, which is how a case is shown to reach the branch it names.  Expected
points come from the oracle's C port (oracle.cref.scalar_mul) or the Python oracle, never from the kernels under test.  Outputs
are compared limb for limb; a failure names the group, the family, the case, the index and the scalar."""
import random

import numpy as np

from oracle import cref
from oracle import oracle as O
from tests import lagrange_ref as LR

# the thirteen groups in the engine's id order
GROUPS = ("bn254_g1", "bn254_g2", "bls12381_g1", "bls12381_g2", "bls12377_g1", "bls12377_g2", "secp256k1_g1", "bw6761_g1",
          "bw6761_g2", "bls24315_g1", "bls24317_g1", "bw6633_g1", "bw6633_g2")
CURVES = LR.CURVES
SCALE_M = 8               # points per thread of k_scale_powers
WIDTHS = (3, 4, 5)        # the ladder's window widths: scale_w, lag_w and the GMSM_SCALE_W / GMSM_LAG_W variant builds
CALL_POINTS = 2 * SCALE_M + 3
GEOMETRIC = ("1,2", "-1,2", "1,1/2", "-2,1", "-2,-1")   # (c, r) of family A, "-x" standing for r - x


def group(name: str) -> O.Group:
    return O.GROUPS[name]


def lag_w(name: str) -> int:
    """the window of k_lag_stage / k_lag_finish (lag_w in lagrange_kernels.cuh)"""
    return 5 if group(name).fr.bits > 300 else 4


def scale_w(name: str) -> int:
    """the window of k_scale_powers (scale_w in mpc_kernels.cuh): lag_w for 8-limb coordinates, 5 for every larger one"""
    return lag_w(name) if group(name).aff_words == 8 else 5


def nwin(name: str, W: int) -> int:
    return group(name).fr.bits // W + 1


# ---- the ladder on integers ----
def digit_stream(s: int, W: int, nw: int) -> list:
    """DigitStream (kernels.cuh) with c = W over nw windows: signed digits d_j with s = sum d_j 2^(W j).  Below the top window
    a window value above 2^(W-1) - 1 becomes value - 2^W with a carry (0 with a carry for an all-ones window that meets one);
    the top window never borrows."""
    out, carry, mask, maxd = [], 0, (1 << W) - 1, (1 << (W - 1)) - 1
    for j in range(nw):
        d = (s & mask) + carry
        s >>= W
        if j < nw - 1 and d > maxd:
            out.append(d - (1 << W))
            carry = 1
        else:
            out.append(d)
            carry = 0
    return out


def compose(digits: list, W: int) -> int:
    return sum(d << (W * j) for j, d in enumerate(digits))


def ladder_additions(s: int, W: int, nw: int, q: int) -> list:
    """the additions acc + (+-table entry) of lag_scalar_mul's Horner loop, as (window, branch) on discrete logarithms mod q
    (the point is [1]): branch "double" when acc == entry (xyzz_add's P == Q case), "cancel" when acc == -entry, "inf" when acc is
    infinity, else "add".  The table's own additions ([k]P + P) are not listed."""
    ds = digit_stream(s, W, nw)
    j = nw - 1
    while j >= 0 and ds[j] == 0:
        j -= 1
    if j < 0:
        return []
    acc, out = ds[j] % q, []
    for j in range(j - 1, -1, -1):
        acc = (acc << W) % q
        if ds[j]:
            e = ds[j] % q
            out.append((j, "inf" if acc == 0 else "double" if acc == e else "cancel" if (acc + e) % q == 0 else "add"))
            acc = (acc + e) % q
    assert acc == s % q
    return out


def digit_cases(name: str, W: int) -> list:
    """the digit-built scalars of family A for window W: (case, s, planned digits or None) with 0 < s < r.  Planned digits lie in
    [-2^(W-1), 2^(W-1) - 1] below the top window and in [0, 2^(W-1)] at the top; digit_stream(s) must give them back exactly.
    Named values (r - 1, ..., 2^W - 1) carry None: they are what they are."""
    q = group(name).fr.q
    nw = nwin(name, W)
    lo, hi, top_hi = -(1 << (W - 1)), (1 << (W - 1)) - 1, 1 << (W - 1)
    out = []

    def planned(case, below, top=None):
        """below: the nw - 1 lower digits; top: the top digit, or the smallest one in [0, 2^(W-1)] putting s in (0, r)"""
        for t in ([top] if top is not None else range(top_hi + 1)):
            ds = list(below) + [t]
            s = compose(ds, W)
            if 0 < s < q:
                out.append((case, s, ds))
                return

    planned("all-min", [lo] * (nw - 1))
    planned("all-max", [hi] * (nw - 1))
    planned("alt-min-max", [lo if j % 2 == 0 else hi for j in range(nw - 1)])
    planned("alt-max-min", [hi if j % 2 == 0 else lo for j in range(nw - 1)])
    for j in range(nw - 1):
        for d in (1, -1, lo):
            below = [0] * (nw - 1)
            below[j] = d
            if d < 0:                  # a negative digit needs a carry above it
                if j + 1 < nw - 1:
                    below[j + 1] = 1
                    planned("single %+d at %d" % (d, j), below, 0)
                else:
                    planned("single %+d at %d" % (d, j), below, 1)
            else:
                planned("single %+d at %d" % (d, j), below, 0)
    for d in (1, top_hi):
        planned("top %d" % d, [0] * (nw - 1), d)
    for t in range(top_hi, 0, -1):      # the largest top digit the bit length allows, lower digits at their minimum
        n0 = len(out)
        planned("top max %d" % t, [lo] * (nw - 1), t)
        if len(out) > n0:
            break
    named = [("r-1", q - 1), ("r-2", q - 2), ("r-3", q - 3), ("(r-1)/2", (q - 1) // 2), ("(r+1)/2", (q + 1) // 2),
             ("2^(W-1)", 1 << (W - 1)), ("2^(W-1)+1", (1 << (W - 1)) + 1), ("2^W-1", (1 << W) - 1)]
    out += [(c, s, None) for c, s in named]
    return out


def geometric(name: str, fam: str) -> tuple:
    """(c, r, n) of a geometric family: out[i] = [c r^i] P_i for i < n = fr.Bits + 40"""
    q = group(name).fr.q
    val = {"1": 1, "2": 2, "-1": q - 1, "-2": q - 2, "1/2": pow(2, -1, q)}
    c, r = (val[x] for x in fam.split(","))
    return c, r, group(name).fr.bits + 40


def geometric_scalars(q: int, c: int, r: int, n: int) -> list:
    out, s = [], c % q
    for _ in range(n):
        out.append(s)
        s = s * r % q
    return out


# ---- points and expected values ----
def gen_enc(name: str) -> np.ndarray:
    G = group(name)
    return G.encode_affine([G.gen])[0]


def random_points(name: str, m: int, seed: int) -> tuple:
    """m random subgroup points [k_i]G from the C port: (discrete logs, (m, words) array)"""
    q = group(name).fr.q
    rng = random.Random(seed)
    ks = [rng.randrange(1, q) for _ in range(m)]
    g = gen_enc(name)
    return ks, np.stack([cref.scalar_mul(name, g, k) for k in ks])


def with_infinity(pts: np.ndarray, ks: list, pos: int) -> tuple:
    """a copy of the points with infinity at pos"""
    pts, ks = pts.copy(), list(ks)
    pts[pos] = 0
    ks[pos] = 0
    return pts, ks


def expected_scaled(job) -> np.ndarray:
    """[s_i] P_i by the C port; job = (name, (m, words) points, scalars); infinity in, or s = 0, gives infinity"""
    name, pts, ss = job
    q = group(name).fr.q
    out = np.zeros_like(pts)
    for i, s in enumerate(ss):
        if pts[i].any() and s % q:
            out[i] = cref.scalar_mul(name, pts[i], s % q)
    return out


def expected_multiples(job) -> np.ndarray:
    """[k_i]G by the C port; job = (name, discrete logs)"""
    name, ks = job
    q = group(name).fr.q
    g = gen_enc(name)
    out = np.zeros((len(ks), group(name).aff_words), dtype=np.uint64)
    for i, k in enumerate(ks):
        if k % q:
            out[i] = cref.scalar_mul(name, g, k % q)
    return out


def compare(what: str, got, want, scalars=None, index=None):
    """limb-exact comparison of (m, words) arrays; names the first wrong index (index[i] for sampled rows) and its scalar"""
    got = np.asarray(got, dtype=np.uint64).reshape(np.shape(want))
    if np.array_equal(got, want):
        return
    i = int(np.nonzero((got != want).any(axis=1))[0][0])
    wrong = int((got != want).any(axis=1).sum())
    sc = "" if scalars is None else ", scalar %d" % scalars[i]
    raise AssertionError("%s: %d wrong points, first at index %d%s\n got  %s\n want %s" % (
        what, wrong, i if index is None else index[i], sc, " ".join("%016x" % int(v) for v in got[i]), " ".join("%016x" % int(v) for v in want[i])))


# ---- family B: every infinity mask of a thread's shared inversion ----
MASK_THREADS = 256
MASK_N = MASK_THREADS * SCALE_M + 5


def mask_layout() -> list:
    """True where point i is infinity: thread t < 256 carries infinity mask t over its 8 points; a tail of 5 finite points"""
    return [i < MASK_THREADS * SCALE_M and bool(((i // SCALE_M) >> (i % SCALE_M)) & 1) for i in range(MASK_N)]


def mask_logs(name: str, c: int, r: int) -> tuple:
    """(input logs, output logs) of family B: input [i + 1]G with the masked points at infinity, output [(i + 1) c r^i]G"""
    q = group(name).fr.q
    inf = mask_layout()
    ks_in = [0 if inf[i] else i + 1 for i in range(MASK_N)]
    sc = geometric_scalars(q, c, r, MASK_N)
    return ks_in, [k * s % q for k, s in zip(ks_in, sc)]


# ---- family C: planted butterflies at every stage of ToLagrangeG1 ----
PLANT_CASES = ("equal", "opposite", "inf-a", "inf-b", "inf-both")


def stage_twiddles(curve: str, n: int, s: int) -> list:
    """w^(-j 2^s) of stage s for j < h = n >> (s + 1) (1 for j = 0)"""
    w_inv, _ = LR.domain_inverses(curve, n)
    q = LR.fr_modulus(curve)
    t = pow(w_inv, 1 << s, q)
    return geometric_scalars(q, 1, t, n >> (s + 1))


def stage_forward(curve: str, x: list, s: int) -> list:
    """stage s of k_lag_stage on discrete logs: blocks of 2h, h = n >> (s + 1), (a, b) -> (a + b, t (a - b)), t = w^(-j 2^s)"""
    q = LR.fr_modulus(curve)
    n = len(x)
    h = n >> (s + 1)
    tw = stage_twiddles(curve, n, s)
    x = list(x)
    for i0 in range(n):
        j = i0 % (2 * h)
        if j < h:
            a, b = x[i0], x[i0 + h]
            x[i0], x[i0 + h] = (a + b) % q, (a - b) * tw[j] % q
    return x


def stage_inverse(curve: str, x: list, s: int) -> list:
    """the inverse of stage_forward: a' = (a + b / t) / 2, b' = (a - b / t) / 2"""
    q = LR.fr_modulus(curve)
    n = len(x)
    h = n >> (s + 1)
    half = pow(2, -1, q)
    tw_inv = [pow(t, -1, q) for t in stage_twiddles(curve, n, s)]
    x = list(x)
    for i0 in range(n):
        j = i0 % (2 * h)
        if j < h:
            a, bt = x[i0], x[i0 + h] * tw_inv[j] % q
            x[i0], x[i0 + h] = (a + bt) * half % q, (a - bt) * half % q
    return x


def plant_positions(n: int, s: int) -> list:
    """the butterflies of stage s that the plan uses: j = 0, 1 and h - 1 of their block (deduplicated for small h)"""
    h = n >> (s + 1)
    return sorted({0, min(1, h - 1), h - 1})


def plant_plan(n: int, s: int) -> list:
    """transforms for stage s: each a list of (case, block, j), every case at every j of plant_positions in a separate butterfly
    (stage s has 2^s blocks, so the early stages need several transforms)"""
    blocks = 1 << s
    todo = [(c, j) for c in PLANT_CASES for j in plant_positions(n, s)]
    out = []
    while todo:
        used, tr, rest = set(), [], []
        for c, j in todo:
            b = next((b for b in range(blocks) if (b, j) not in used), None)
            if b is None:
                rest.append((c, j))
            else:
                used.add((b, j))
                tr.append((c, b, j))
        out.append(tr)
        todo = rest
    return out


def planted_logs(curve: str, n: int, s: int, plan: list, seed: int) -> list:
    """input discrete logs whose state at the start of stage s holds the planted butterflies of `plan` (random non-zero values
    elsewhere); checked by running stages 0 .. s - 1 forward again"""
    q = LR.fr_modulus(curve)
    rng = random.Random(seed)
    h = n >> (s + 1)
    x = [rng.randrange(1, q) for _ in range(n)]
    for case, b, j in plan:
        i0, k = 2 * h * b + j, rng.randrange(1, q)
        x[i0], x[i0 + h] = {"equal": (k, k), "opposite": (k, q - k), "inf-a": (0, k), "inf-b": (k, 0), "inf-both": (0, 0)}[case]
    state = x
    for t in range(s - 1, -1, -1):
        x = stage_inverse(curve, x, t)
    check_planted(curve, x, s, plan, state)
    return x


def check_planted(curve: str, logs: list, s: int, plan: list, state: list):
    q = LR.fr_modulus(curve)
    n = len(logs)
    h = n >> (s + 1)
    y = logs
    for t in range(s):
        y = stage_forward(curve, y, t)
    assert y == state, (curve, n, s, "the inverse stages do not invert the forward ones")
    for case, b, j in plan:
        a, bb = y[2 * h * b + j], y[2 * h * b + j + h]
        ok = {"equal": a == bb and a != 0, "opposite": a != 0 and (a + bb) % q == 0, "inf-a": a == 0 and bb != 0,
              "inf-b": a != 0 and bb == 0, "inf-both": a == 0 and bb == 0}[case]
        assert ok, (curve, n, s, case, b, j, a, bb)


def planted_transforms(curve: str, n: int, seed: int) -> list:
    """(stage, plan, input logs) for every stage of a transform of n points"""
    out = []
    logn = n.bit_length() - 1
    for s in range(logn):
        for k, plan in enumerate(plant_plan(n, s)):
            out.append((s, plan, planted_logs(curve, n, s, plan, seed + 1000 * s + k)))
    return out


def lagrange_points_ref(job) -> np.ndarray:
    """lagrange_ref.to_lagrange_g1 (the point-domain restatement) on [logs]G; job = (curve, logs)"""
    curve, logs = job
    G = LR.group(curve)
    pts = [G.scalar_mul(G.gen, k) if k else G.aff_inf() for k in logs]
    return G.encode_affine(LR.to_lagrange_g1(curve, pts))


def plan_text(plan: list) -> str:
    return ", ".join("%s at block %d j %d" % c for c in plan)


# ---- family D: the ramp [i + 1]G ----
def ramp_lagrange(curve: str, n: int, idx) -> list:
    """discrete logs of ToLagrangeG1([1]G, [2]G, ..., [n]G) at the indices idx: (n + 1) / 2 at 0, 1 / (w^(-j) - 1) elsewhere"""
    q = LR.fr_modulus(curve)
    w_inv, _ = LR.domain_inverses(curve, n)
    return [(n + 1) * pow(2, -1, q) % q if j == 0 else pow(pow(w_inv, j, q) - 1, -1, q) for j in idx]


def sample_indices(n: int, seed: int, m: int = 4096) -> list:
    """0, 1, n/2 +- 1, n - 2, n - 1, every 2^k and 2^k +- 1, then random indices up to m in all"""
    idx = {0, 1, n // 2 - 1, n // 2, n // 2 + 1, n - 2, n - 1}
    k = 1
    while k < n:
        idx |= {k - 1, k, k + 1}
        k <<= 1
    idx = {i for i in idx if 0 <= i < n}
    rng = random.Random(seed)
    while len(idx) < min(m, n):
        idx.add(rng.randrange(n))
    return sorted(idx)


def monomial_indices(n: int, seed: int) -> list:
    """0, 7, 8, 9, every 2^k - 1, 2^k, 2^k + 1, the last 64 and 4096 random indices below n"""
    idx = {0, 7, 8, 9} | set(range(max(0, n - 64), n))
    k = 1
    while k < n:
        idx |= {k - 1, k, k + 1}
        k <<= 1
    rng = random.Random(seed)
    idx |= {rng.randrange(n) for _ in range(4096)}
    return sorted(i for i in idx if 0 <= i < n)
