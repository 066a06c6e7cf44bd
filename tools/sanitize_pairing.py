"""small calls of every pairing entry (MillerLoop, FinalExponentiation, Pair; host and device), for compute-sanitizer:
   compute-sanitizer --tool memcheck python tools/sanitize_pairing.py"""
import importlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
importlib.import_module("gnark_crypto_b200")
pr = importlib.import_module("gnark-crypto_b200.pairing")
from tests import pairing_cases as PC  # noqa: E402
from tests import pairing_ref as PR  # noqa: E402

ok = True
for curve in ("bn254", "bls12381"):
    T = PR.tower(curve)
    P, Q = PC.random_pairs(curve, 5, seed=9)
    P[2] = T.G1.aff_inf()
    pa, qa = PC.encode_pairs(curve, P, Q)
    ml = T.miller_loop(P, Q)
    ok = ok and np.array_equal(pr.MillerLoop(curve, pa, qa).reshape(1, -1), T.encode([ml]))
    ok = ok and np.array_equal(pr.Pair(curve, pa, qa).reshape(1, -1), T.encode([T.final_exp(ml)]))
    z = T.encode([ml, T.one()])
    ok = ok and np.array_equal(pr.FinalExponentiation(curve, z[0], z[1]).reshape(1, -1), T.encode([T.final_exp(ml)]))
print("sanitize_pairing:", "ok" if ok else "MISMATCH")
sys.exit(0 if ok else 1)
