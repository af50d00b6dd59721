"""Build libb200gnss.so in-tree with nvcc for sm_90a (H100) (no JIT cache, no torch extension).

    python -m gnss_sdr_b200.build [--force] [--verbose] [--ptxas] [-DNAME=VALUE ...] [--out=PATH]

A build is redone when its inputs change: the name and bytes of every file in csrc/ and of include/b200gnss.h, and every
nvcc flag.  Their hash is stamped beside the output (<output>.srchash).  File times play no part, since a tree copied to
another machine keeps its contents but not necessarily its mtimes.
"""
from __future__ import annotations

import hashlib
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
HEADER = os.path.join(os.path.dirname(HERE), "include", "b200gnss.h")
OBJ_DIR = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libb200gnss.so")
VARIANTS = os.path.join(HERE, "variants")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC,-O3,-Wall",
    "--expt-relaxed-constexpr",
    "-cudart", "static",
]
LINK_FLAGS = ["-cudart", "static", "-Xlinker", "--no-undefined"]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def compile_flags(src, extra=()):
    # *_nofma.cu: host-parity arithmetic (DLL/PLL loop) - every multiply and add rounds separately
    return FLAGS + (["--fmad=false"] if src.endswith("_nofma.cu") else []) + list(extra)


def input_hash(extra=()) -> str:
    """hash of everything a build's output depends on: csrc/ and the header (names and bytes) and the nvcc flags"""
    h = hashlib.sha256()
    for path in sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC)) + [HEADER]:
        with open(path, "rb") as fh:
            data = fh.read()
        h.update(f"{os.path.basename(path)} {len(data)}\n".encode())
        h.update(data)
    flags = {os.path.basename(src): compile_flags(src, extra) for src in sources()}
    h.update(json.dumps([flags, LINK_FLAGS], sort_keys=True).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False, ptxas_v: bool = False, extra=(), out: str = None) -> str:
    """extra: additional nvcc flags (e.g. -DSH_STAGES=8) and out: alternative output path, for A/B variants."""
    out = out or LIB
    want = input_hash(extra)
    stamp = out + ".srchash"
    if not force and os.path.exists(out) and os.path.exists(stamp):
        with open(stamp) as fh:
            if fh.read().strip() == want:
                return out
    objs = []
    os.makedirs(OBJ_DIR, exist_ok=True)
    procs = []
    for src in sources():
        obj = os.path.join(OBJ_DIR, os.path.basename(src)[:-3] + ("" if out == LIB else "_" + os.path.basename(out)) + ".o")
        cmd = [NVCC] + compile_flags(src, extra) + (["-Xptxas", "-v"] if ptxas_v else []) + ["-c", src, "-o", obj]
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
    cmd = [NVCC, "-shared", "-o", out] + objs + LINK_FLAGS
    if verbose:
        print(" ".join(cmd), flush=True)
    subprocess.check_call(cmd)
    with open(stamp, "w") as fh:
        fh.write(want + "\n")
    return out


def build_variant(stages: int, stress: bool) -> str:
    """The same sources with -DSH_STAGES=stages -DSH_STRESS=0|1 (the TMA ring's depth, and pseudo-random delays injected
    into its producer and consumers), into variants/libb200gnss_ring<stages>_<stress|plain>.so."""
    os.makedirs(VARIANTS, exist_ok=True)
    out = os.path.join(VARIANTS, f"libb200gnss_ring{stages}_{'stress' if stress else 'plain'}.so")
    return build(extra=[f"-DSH_STAGES={stages}", f"-DSH_STRESS={1 if stress else 0}"], out=out)


if __name__ == "__main__":
    extra = [a for a in sys.argv[1:] if a.startswith("-D")]
    outs = [a.split("=", 1)[1] for a in sys.argv[1:] if a.startswith("--out=")]
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv, ptxas_v="--ptxas" in sys.argv, extra=extra,
                out=outs[0] if outs else None))
