"""Big-int restatement of the point updates and linear combinations of mpcsetup (ecc/bn254/mpcsetup/mpcsetup.go; the mpcsetup
packages of the other pairing curves are the same generated code) on the oracle's group operations (TEST INFRASTRUCTURE).

  * `scale_powers`: A[i] <- [c r^i] A[i], one scalar multiplication per point (the slice loop of UpdateValues, :64-81, for r = 1;
    UpdateMonomials for c = r on A[1:]);
  * `update_monomials`: UpdateMonomialsG1 / G2 (:365-381) step by step, A[i] <- [r^i] A[i] for i >= 1;
  * `linear_combinations`: linearCombinationsG1 / G2 (:396-447, :489-540) line by line on copies of A and powers, with the
    reference's in-place updates (so its results are reproduced whatever `powers` holds, powers[1] = 0 included: the inverse of 0
    is 0 in fr.Element.Inverse).
Points are oracle affine points ((0, 0) = infinity), scalars integers mod r."""
from oracle import oracle as O


def group(name: str) -> O.Group:
    return O.GROUPS[name]


def scale_powers(G: O.Group, pts: list, c: int, r: int) -> list:
    q = G.fr.q
    out, s = [], c % q
    for p in pts:
        out.append(G.scalar_mul(p, s) if s else G.aff_inf())
        s = s * r % q
    return out


def update_monomials(G: O.Group, A: list, r: int) -> list:
    """UpdateMonomialsG1 / G2 on a copy of A: A[1] <- [r]A[1], then A[i] <- [r^i]A[i] (len(A) < 2 raises IndexError, the Go panic)"""
    q = G.fr.q
    A = list(A)
    A[1] = G.scalar_mul(A[1], r % q)
    r_exp = r * r % q
    for i in range(2, len(A)):
        e = r_exp
        if i + 1 != len(A):
            r_exp = r_exp * r % q
        A[i] = G.scalar_mul(A[i], e)
    return A


def _msm(G: O.Group, pts: list, ks: list):
    return O.msm_naive(G, pts, [k % G.fr.q for k in ks])


def linear_combinations(G: O.Group, A: list, powers: list, ends: list):
    """(truncated, shifted) of linearCombinationsG1 / G2; A and powers are not modified"""
    q = G.fr.q
    if ends[-1] != len(A) or len(A) != len(powers):
        raise ValueError("lengths mismatch")
    if len(ends) == 1 and ends[0] == 2:
        return A[0], A[1]
    A, powers = list(A), [p % q for p in powers]
    for e in ends:
        powers[e - 1] = 0
    truncated = _msm(G, A, powers)
    r_inv_neg = (-pow(powers[1], -1, q)) % q if powers[1] else 0
    prev_end = 0
    for i, e in enumerate(ends):
        powers[2 * i] = powers[prev_end] * r_inv_neg % q
        powers[2 * i + 1] = powers[e - 2]
        A[2 * i] = A[prev_end]
        A[2 * i + 1] = A[e - 1]
        prev_end = e
    k = 2 * len(ends)
    powers[k] = (-r_inv_neg) % q
    A[k] = truncated
    shifted = _msm(G, A[: k + 1], powers[: k + 1])
    return truncated, shifted
