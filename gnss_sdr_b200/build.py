"""Build libb200gnss.so in-tree with nvcc for sm_90a (H100) (no JIT cache, no torch extension).

    python -m gnss_sdr_b200.build [--force] [--verbose]
"""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libb200gnss.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC,-O3,-Wall",
    "--expt-relaxed-constexpr",
    "-cudart", "static",
]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "b200gnss.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False, ptxas_v: bool = False, extra=(), out: str = None) -> str:
    """extra: additional nvcc flags (e.g. -DSH_STAGES=8) and out: alternative output path, for A/B variants."""
    if out:
        force = True
    if not force and not needs_build():
        return LIB
    objs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    procs = []
    for src in sources():
        obj = os.path.join(HERE, "build", os.path.basename(src)[:-3] + ".o")
        obj = obj if not out else obj[:-2] + "_" + os.path.basename(out) + ".o"
        # *_nofma.cu: host-parity arithmetic (DLL/PLL loop) - every multiply and add rounds separately
        per_file = ["--fmad=false"] if src.endswith("_nofma.cu") else []
        cmd = [NVCC] + FLAGS + per_file + list(extra) + (["-Xptxas", "-v"] if ptxas_v else []) + ["-c", src, "-o", obj]
        if verbose:
            print(" ".join(cmd), flush=True)
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for src, p in procs:
        txt, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write(txt)
        elif verbose or ptxas_v:
            sys.stdout.write(txt)
    if failed:
        raise RuntimeError("nvcc failed")
    cmd = [NVCC, "-shared", "-o", out or LIB] + objs + ["-cudart", "static", "-Xlinker", "--no-undefined"]
    if verbose:
        print(" ".join(cmd), flush=True)
    subprocess.check_call(cmd)
    return out or LIB


if __name__ == "__main__":
    extra = [a for a in sys.argv[1:] if a.startswith("-D")]
    outs = [a.split("=", 1)[1] for a in sys.argv[1:] if a.startswith("--out=")]
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv, ptxas_v="--ptxas" in sys.argv, extra=extra,
                out=outs[0] if outs else None))
