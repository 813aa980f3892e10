"""Build libbzk.so (sm_90a, H100) in-tree.  `python -m bazuka_b200.build [-f]`.

nvcc cross-compiles without a GPU; the resulting bazuka_b200/libbzk.so is git-ignored and rebuilt
from source by every checkout."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "_obj")
SO = os.path.join(HERE, "libbzk.so")
SOURCES = ["msm_g2.cu", "msm_g1.cu", "groth16.cu", "poseidon.cu", "poseidon_host.cu", "ntt.cu", "verify.cu", "witness.cu", "mpn_host.cu", "mpn_wire.cu", "mpn_prover.cu", "mpn_worker.cu", "mpn_circuit.cu", "params_io.cu", "jubjub.cu", "ed25519.cu", "capi.cu"]
HEADERS = ["ff.cuh", "ec.cuh", "common.cuh", "msm_impl.cuh", "witness_core.cuh", "jubjub.cuh", "pairing.cuh", os.path.join("..", "..", "include", "bzk.h")]
# headers only some sources include
EXTRA_DEPS = {"mpn_wire.cu": ["mpn_wire.cuh"], "mpn_host.cu": ["mpn_wire.cuh", "hash_plan.cuh"], "poseidon.cu": ["hash_plan.cuh"], "mpn_prover.cu": ["mpn_wire.cuh"], "mpn_worker.cu": ["mpn_wire.cuh"], "params_io.cu": ["params_io.cuh"], "groth16.cu": ["r1cs_blocked.cuh"], "jubjub.cu": ["mpn_wire.cuh"], "ed25519.cu": ["ed25519.cuh", "mpn_wire.cuh"]}
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xptxas", "-v",
] + os.environ.get("BZK_NVCC_EXTRA", "").split()   # e.g. BZK_NVCC_EXTRA=-DBZK_MUL_NOINLINE for code-size experiments (use -f)


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    hdrs = [os.path.join(CSRC, h) for h in HEADERS]
    jobs = []
    for s in SOURCES:
        src = os.path.join(CSRC, s)
        obj = os.path.join(OBJ, s.replace(".cu", ".o"))
        if force or _stale(obj, [src] + hdrs + [os.path.join(CSRC, h) for h in EXTRA_DEPS.get(s, [])]):
            jobs.append((src, obj))

    def compile_one(job):
        src, obj = job
        r = subprocess.run([NVCC] + FLAGS + ["-c", src, "-o", obj], capture_output=True, text=True)
        with open(obj + ".log", "w") as f:
            f.write(r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{r.stdout}\n{r.stderr}")
        return r.stderr

    with ThreadPoolExecutor(max_workers=7) as ex:
        logs = list(ex.map(compile_one, jobs))
    if verbose:
        for l in logs:
            print(l)
    objs = [os.path.join(OBJ, s.replace(".cu", ".o")) for s in SOURCES]
    if force or jobs or _stale(SO, objs):
        r = subprocess.run([NVCC, "-shared", "-o", SO] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"],
                           capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return SO


if __name__ == "__main__":
    print(build(force="-f" in sys.argv, verbose="-v" in sys.argv))
