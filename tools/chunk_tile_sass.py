"""Count the chunk path's interior tile in SASS: instructions, shared-memory wavefronts and the issue / pipe estimate.

    python tools/chunk_tile_sass.py

Compiles tools/chunk_tile_probe.cu (warp_tile_chunks alone in a loop, the kernel's launch bounds) and trk_shared_kernel.cu
for sm_90a with -Xptxas -v, and needs no GPU.  For each tap count it prints the loop body's instructions by opcode and
the estimate per tile and warp:

    issue  = instructions / 4          (four schedulers per SM, one instruction each per cycle)
    pipe   = shared-memory wavefronts  (one 128-byte wavefront per cycle per SM)

Wavefronts per instruction, by the access pattern of warp_tile_chunks (the model, not a measurement):
    LDS.128  the first 8 are the lane's samples, 512 B conflict-free: 4 each; the others read D^j, a broadcast: 1 each
    STS.128  (a running-sum scratch, 144-byte lane stride, conflict-free): 4 each
    LDS.64   (a running sum read back at a lane-dependent index): 3 each (2 to 4)
    LDS      a code value; the lanes of a warp read about 24 neighbouring chips: 1.25 each
plus 4 per tile for the producer's TMA writes of the tile (4 KB), which every consumer warp's share of the pipe carries.
The loop body also holds the probe's own per-tile work (z0 advance, slot address, loop test): about 10 instructions that
the kernel spends too, beside its ring waits and arrivals.
Then the register and spill lines of trk_shared_kernel<1|3|5> from ptxas.
"""
from __future__ import annotations

import os
import re
import subprocess
import sys
import tempfile
from collections import Counter

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gnss_sdr_b200.build import NVCC  # noqa: E402

CUOBJDUMP = os.path.join(os.path.dirname(NVCC), "cuobjdump")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-Xptxas", "-v", "-cubin"]
WAVES = {"LDS.128": None, "STS.128": 4.0, "LDS.64": 3.0, "LDS": 1.25}
TMA_WAVES = 4.0


def compile_cubin(src, out):
    p = subprocess.run([NVCC] + FLAGS + ["-o", out, src], capture_output=True, text=True)
    if p.returncode != 0:
        sys.stderr.write(p.stdout + p.stderr)
        raise SystemExit("nvcc failed")
    return p.stdout + p.stderr


def ptxas_resources(log):
    """{mangled name: (registers, spill stores, spill loads)}"""
    res, name, spill = {}, None, (0, 0)
    for line in log.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            name = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            spill = (int(m.group(1)), int(m.group(2)))
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            name = m.group(1)
        m = re.search(r"Used (\d+) registers", line)
        if m and name:
            res[name] = (int(m.group(1)),) + spill
            spill = (0, 0)
    return res


def sass_functions(cubin):
    txt = subprocess.run([CUOBJDUMP, "-sass", cubin], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in txt.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = funcs.setdefault(m.group(1), [])
            continue
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?);", line)
        if m and cur is not None:
            cur.append((int(m.group(1), 16), m.group(2).strip()))
    return funcs


def opcode(ins):
    ins = re.sub(r"^@!?U?P[T0-9]+\s+", "", ins)
    return ins.split()[0]


def loop_body(code):
    """instructions of the largest loop: from the target of a backward branch to the branch"""
    best = []
    for i, (addr, ins) in enumerate(code):
        m = re.match(r"(?:@!?U?P\d\s+)?BRA\s+(?:`\()?\S*?0x([0-9a-f]+)", ins)
        if m and int(m.group(1), 16) < addr:
            tgt = int(m.group(1), 16)
            body = [c for c in code if tgt <= c[0] <= addr]
            if len(body) > len(best):
                best = body
    return [ins for _, ins in best if opcode(ins) != "NOP"]


def tally(body):
    ops = Counter(opcode(i) for i in body)
    waves, lds128 = TMA_WAVES, 0
    for op, n in ops.items():
        if op == "LDS.128":
            samples = min(n, 8)
            waves += 4.0 * samples + 1.0 * (n - samples)
            lds128 = n
        elif op in WAVES:
            waves += WAVES[op] * n
        elif op.startswith("LDS.U") or op.startswith("LDS.S"):
            waves += 1.25 * n
    return ops, waves, lds128


def main():
    with tempfile.TemporaryDirectory() as tmp:
        probe = os.path.join(tmp, "probe.cubin")
        log = compile_cubin(os.path.join(ROOT, "tools", "chunk_tile_probe.cu"), probe)
        funcs = sass_functions(probe)
        res = ptxas_resources(log)
        rows = []
        for name, code in sorted(funcs.items()):
            m = re.search(r"chunk_tile_probeILi(\d)ELb0EE", name)
            if not m:
                continue
            body = loop_body(code)
            ops, waves, _ = tally(body)
            rows.append((int(m.group(1)), len(body), waves, ops, res.get(name)))
        for taps, n, waves, ops, r in sorted(rows):
            print(f"<{taps}> interior tile: {n} instructions, "
                  f"{waves:.0f} wavefronts -> issue {n / 4:.0f}, pipe {waves:.0f}, max {max(n / 4, waves):.0f} cycles per tile and warp"
                  + (f"  (probe: {r[0]} registers, spills {r[1]} / {r[2]} B)" if r else ""))
            print("    " + ", ".join(f"{k} {v}" for k, v in sorted(ops.items(), key=lambda kv: (-kv[1], kv[0]))))
        kern = os.path.join(tmp, "kernel.cubin")
        log = compile_cubin(os.path.join(ROOT, "gnss_sdr_b200", "csrc", "trk_shared_kernel.cu"), kern)
        for name, (regs, st, ld) in sorted(ptxas_resources(log).items()):
            m = re.search(r"trk_shared_kernelILi(\d)E", name)
            if m:
                print(f"trk_shared_kernel<{m.group(1)}>: {regs} registers, spill stores {st} B, spill loads {ld} B")


if __name__ == "__main__":
    main()
