"""Build libdfold_b200.so (sm_90a) in-tree with nvcc.  Used by __graft_entry__.build() and `python -m dynamicpdb_b200.build`."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libdfold_b200.so")
SOURCES = ["simt.cu", "rigid.cu", "epilogue.cu", "diffuse.cu", "metrics.cu", "rollout.cu", "loss.cu", "aux_loss.cu", "featurize.cu", "ipa_attn.cu", "ipa_v2.cu", "ipa_fused.cu", "gemm_sm90.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
         "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    objs = []
    procs = []
    for s in SOURCES:
        o = os.path.join(CSRC, s.replace(".cu", ".o"))
        objs.append(o)
        cmd = [NVCC, *FLAGS, "-c", os.path.join(CSRC, s), "-o", o] + (["-Xptxas", "-v"] if verbose else [])
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    ok = True
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            ok = False
            sys.stderr.write(f"[dfold build] {s} failed:\n{out}\n")
        elif verbose or out.strip():
            sys.stderr.write(f"[dfold build] {s}:\n{out}\n")
    if not ok:
        raise RuntimeError("nvcc failed")
    subprocess.check_call([NVCC, *FLAGS[:2], "-shared", "-o", LIB, *objs, "-cudart", "static"])
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
