"""In-tree build of libgmsm.so (sm_90a) -- `python gnark-crypto_b200/build.py [-f]`.

Each (curve, group) instantiation is its own translation unit (csrc/inst_*.cu) so the heavy
ptxas work runs in parallel; objects are cached by source mtime under build/."""
import concurrent.futures as cf
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
# GMSM_BUILD_TAG=<tag> builds an experimental variant into build_<tag>/ and libgmsm_<tag>.so (loaded with
# GMSM_LIB=<tag>); extra nvcc flags for it come from GMSM_NVCC_EXTRA
TAG = os.environ.get("GMSM_BUILD_TAG", "")
BUILD = os.path.join(HERE, "build" + ("_" + TAG if TAG else ""))
LIB = os.path.join(HERE, "libgmsm%s.so" % ("_" + TAG if TAG else ""))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
    "-Xcompiler", "-fPIC", "-Xptxas", "-v",
]
UNITS = ["gmsm.cu", "fft.cu", "decode.cu", "pairing.cu", "inst_bn254_g1.cu", "inst_bn254_g2.cu", "inst_bls12381_g1.cu", "inst_bls12381_g2.cu", "inst_bls12377_g1.cu", "inst_bls12377_g2.cu",
         "inst_secp256k1_g1.cu", "inst_bw6761_g1.cu", "inst_bw6761_g2.cu",
         "inst_bls24315_g1.cu", "inst_bls24317_g1.cu", "inst_bw6633_g1.cu", "inst_bw6633_g2.cu"]


def _newest_dep():
    deps = glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(CSRC, "*.h")) + [
        os.path.join(HERE, "..", "include", "gmsm.h")
    ]
    return max(os.path.getmtime(d) for d in deps)


def _compile(unit, force):
    src = os.path.join(CSRC, unit)
    obj = os.path.join(BUILD, unit.replace(".cu", ".o"))
    log = obj + ".log"
    if not force and os.path.exists(obj) and os.path.getmtime(obj) > max(os.path.getmtime(src), _newest_dep()):
        return unit, 0, "cached"
    extra = os.environ.get("GMSM_NVCC_EXTRA", "").split()
    cmd = [NVCC] + FLAGS + extra + ["-c", src, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    open(log, "w").write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
    return unit, r.returncode, r.stderr if r.returncode else "built"


def build(force=False, verbose=True):
    os.makedirs(BUILD, exist_ok=True)
    with cf.ThreadPoolExecutor(max_workers=len(UNITS)) as ex:
        res = list(ex.map(lambda u: _compile(u, force), UNITS))
    for unit, rc, msg in res:
        if verbose:
            print("[build] %-24s %s" % (unit, msg if rc == 0 else "FAILED"))
        if rc != 0:
            raise RuntimeError("nvcc failed for %s:\n%s" % (unit, msg))
    objs = [os.path.join(BUILD, u.replace(".cu", ".o")) for u in UNITS]
    if force or not os.path.exists(LIB) or any(os.path.getmtime(o) > os.path.getmtime(LIB) for o in objs):
        cmd = [NVCC, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n" + r.stdout + r.stderr)
        if verbose:
            print("[build] linked", LIB)
    return LIB


if __name__ == "__main__":
    build(force="-f" in sys.argv)
