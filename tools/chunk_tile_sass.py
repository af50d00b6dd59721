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
The probe's loop is counted along the path one interior tile takes when the first and the last tap share their
running-sum pick (the shortest path through the loop that reads the tile), and again along the path that runs the last
tap's own select tree.
Then the kernel itself: the chunk path's tile loop of trk_shared_kernel<1|3|5> (the loop that waits on the ring, arrives
on it and holds the most FSEL), counted along the same two paths, so that the ring walk around the tile is in the count:
an interior tile that does not re-seed its phasor.  And the register and spill lines of trk_shared_kernel<1|3|5> from
ptxas.
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


BRANCH = re.compile(r"(?:@!?U?P\w+\s+)?BRA(?:\.\w+)*\s+(?:!?U?P\w+,\s+)?(?:`\()?\S*?0x([0-9a-f]+)")


def branch_target(ins):
    m = BRANCH.match(ins)
    return int(m.group(1), 16) if m else None


def loops(code):
    """(first, last) instruction indices of every loop closed by a predicated backward branch (an unconditional one
    jumps back from an out-of-line retry or divergence stub)"""
    at = {a: i for i, (a, _) in enumerate(code)}
    return [(at[t], i) for i, (a, ins) in enumerate(code)
            if ins.startswith("@") and (t := branch_target(ins)) is not None and t < a and t in at]


def shortest_path(code, first, last, need):
    """fewest instructions (NOPs not counted) from code[first] to code[last] over forward edges, among the paths on which
    each opcode in `need` occurs at least need[op] times; None when no path does.  Branches out of [first, last] (retry
    and divergence stubs) count as not taken."""
    ops = sorted(need)
    goal = tuple(need[o] for o in ops)
    at = {a: i for i, (a, _) in enumerate(code)}
    best = {first: {(0,) * len(ops): (0, None)}}
    for i in range(first, last + 1):
        states = best.get(i)
        if not states:
            continue
        ins = code[i][1]
        op = opcode(ins)
        cost = 0 if op == "NOP" else 1
        cond = ins.startswith("@") or re.match(r"BRA(?:\.\w+)*\s+!?U?P\w+,", ins) is not None
        succ = []
        if op.startswith("BRA") and op != "BRA.DIV" and "ANY" not in op:
            t = branch_target(ins)
            if t is not None and code[i][0] < t <= code[last][0]:
                succ.append(at[t])
            if cond:
                succ.append(i + 1)
        elif not (op == "EXIT" and not cond):
            succ.append(i + 1)
        for key, (n, _) in states.items():
            k2 = tuple(min(need[o], c + (op == o)) for o, c in zip(ops, key))
            for j in succ:
                if j <= last:
                    d = best.setdefault(j, {})
                    if k2 not in d or d[k2][0] > n + cost:
                        d[k2] = (n + cost, (i, key))
    if goal not in best.get(last, {}):
        return None
    path, i, key = [], last, goal
    while True:
        path.append(code[i][1])
        prev = best[i][key][1]
        if prev is None:
            break
        i, key = prev
    return [ins for ins in reversed(path) if opcode(ins) != "NOP"]


def tile_paths(code, first, last, taps):
    """the shared-pick path (shortest through the 16 LDS.128 of a tile) and, for 3 taps (the only count that pairs its
    taps), the path with the last tap's own select tree (20 FSEL more)"""
    shared = shortest_path(code, first, last, {"LDS.128": 16})
    fsel = sum(opcode(i) == "FSEL" for i in shared)
    return shared, shortest_path(code, first, last, {"LDS.128": 16, "FSEL": fsel + 20}) if taps == 3 else None


def kernel_chunk_loop(code):
    """the chunk path's tile loop: waits on and arrives at the ring, most FSEL"""
    cands = [(f, l) for f, l in loops(code) if any("TRYWAIT" in c[1] for c in code[f:l + 1])
             and any("SYNCS.ARRIVE" in c[1] for c in code[f:l + 1])]
    return max(cands, key=lambda fl: sum(opcode(c[1]) == "FSEL" for c in code[fl[0]:fl[1] + 1]))


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
            first, last = max(loops(code), key=lambda fl: fl[1] - fl[0])
            body, own = tile_paths(code, first, last, int(m.group(1)))
            ops, waves, _ = tally(body)
            rows.append((int(m.group(1)), len(body), len(own) if own else None, waves, ops, res.get(name)))
        for taps, n, n_own, waves, ops, r in sorted(rows):
            print(f"<{taps}> interior tile: {n} instructions" + (f" (own pick for the last tap: {n_own})" if n_own else "") + ", "
                  f"{waves:.0f} wavefronts -> issue {n / 4:.0f}, pipe {waves:.0f}, max {max(n / 4, waves):.0f} cycles per tile and warp"
                  + (f"  (probe: {r[0]} registers, spills {r[1]} / {r[2]} B)" if r else ""))
            print("    " + ", ".join(f"{k} {v}" for k, v in sorted(ops.items(), key=lambda kv: (-kv[1], kv[0]))))
        kern = os.path.join(tmp, "kernel.cubin")
        log = compile_cubin(os.path.join(ROOT, "gnss_sdr_b200", "csrc", "trk_shared_kernel.cu"), kern)
        for name, code in sorted(sass_functions(kern).items()):
            m = re.search(r"trk_shared_kernelILi(\d)E", name)
            if not m:
                continue
            body, own = tile_paths(code, *kernel_chunk_loop(code), int(m.group(1)))
            print(f"trk_shared_kernel<{m.group(1)}> chunk-path tile loop, interior tile without re-seed: {len(body)} instructions"
                  + (f" (own pick for the last tap: {len(own)})" if own else ""))
            print("    " + ", ".join(f"{k} {v}" for k, v in Counter(opcode(i) for i in body).most_common()))
        for name, (regs, st, ld) in sorted(ptxas_resources(log).items()):
            m = re.search(r"trk_shared_kernelILi(\d)E", name)
            if m:
                print(f"trk_shared_kernel<{m.group(1)}>: {regs} registers, spill stores {st} B, spill loads {ld} B")


if __name__ == "__main__":
    main()
