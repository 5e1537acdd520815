#!/usr/bin/env python
"""Instruction counts of the hot blocks of the batch march kernel, read from its SASS (no GPU needed).

Compiles volrend_b200/csrc/vr_kernels_inst.cu for sm_90a to a cubin (one per basis size), disassembles the product
batch kernel march_persistent_kernel<KBD, false, kOutLinear> with cuobjdump and splits its march loop:

  march loop   the innermost loop that contains the colour-record loads (LDG.E.128.CONSTANT)
  fetch loop   the loop nested in it: one more table fetch of find_leaf_wide
  shading      the forward branch of the march loop that skips the record loads (sigma > sigma_thresh): the
               expf / weight, the record fetch and the colour of one shaded sample.  "common" leaves out the
               division slow paths (a predicated branch around a CALL), which the bench never takes.
  body         the rest of the march loop, minus the fetch loop's exit block: what an empty sample whose leaf
               is found by the first fetch executes.

Prints the counts, the kernel's registers and spills (ptxas -v), and the lane_sim.c cost constants they give.

    python tools/sass_blocks.py                 # KBD 16 and 25, this tree
    python tools/sass_blocks.py --src OTHER     # another checkout (e.g. the parent commit) for a before/after
"""
import argparse
import os
import re
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INST_RE = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;")


def nvcc_path():
    p = shutil.which("nvcc")
    if p:
        return p
    for c in (os.path.join(os.environ.get("CUDA_HOME", ""), "bin", "nvcc"), "/usr/local/cuda/bin/nvcc"):
        if os.path.isfile(c):
            return c
    sys.exit("nvcc not found (set CUDA_HOME or put nvcc on PATH)")


def kernel_names(kbd):
    """Mangled names of the batch kernel: march_persistent_kernel<KBD, false, kOutLinear>, and the same kernel in
    checkouts that still carry the top-grid and tuning parameters (<KBD, false, false, kOutLinear, 193>)."""
    kb = f"Li{kbd}E" if kbd >= 0 else f"Lin{-kbd}E"
    return [f"_ZN3vrb23march_persistent_kernelI{kb}Lb0ELi0EEEvNS_9LaunchDevE",
            f"_ZN3vrb23march_persistent_kernelI{kb}Lb0ELb0ELi0ELi193EEEvNS_9LaunchDevE"]


def compile_cubin(src, kbd, out_dir, extra):
    nvcc = nvcc_path()
    cubin = os.path.join(out_dir, f"vr_kernels_{kbd}.cubin")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
           "-I" + os.path.join(src, "include"), "-I" + os.path.join(src, "volrend_b200", "csrc"),
           "-diag-suppress", "20012", f"-DVR_KBD={kbd}",
           "-Xptxas", "-v", "-cubin", os.path.join(src, "volrend_b200", "csrc", "vr_kernels_inst.cu"), "-o", cubin]
    cmd += extra
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.exit(r.stdout + r.stderr)
    return cubin, r.stderr


def ptxas_stats(log, name):
    """(registers, stack frame bytes, spill store bytes, spill load bytes) of one kernel from ptxas -v."""
    lines = log.splitlines()
    for i, ln in enumerate(lines):
        if f"Function properties for {name}" in ln:
            st = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", lines[i + 1])
            rg = re.search(r"Used (\d+) registers", lines[i + 2])
            return int(rg.group(1)), int(st.group(1)), int(st.group(2)), int(st.group(3))
    sys.exit(f"no ptxas statistics for {name}")


def disassemble(cubin, name):
    cuobjdump = os.path.join(os.path.dirname(nvcc_path()), "cuobjdump")
    r = subprocess.run([cuobjdump, "-sass", "-fun", name, cubin], capture_output=True, text=True, check=True)
    ins = []
    for ln in r.stdout.splitlines():
        m = INST_RE.search(ln)
        if m:
            ins.append((int(m.group(1), 16), m.group(2)))
    if not ins:
        sys.exit(f"{name} not found in {cubin}")
    return ins


def branch_target(text):
    """Target address of a BRA (None for anything else, or an indirect branch)."""
    m = re.match(r"(@!?U?P\w+\s+)?BRA(\.\w+)*\s+(!?U?P\w+,\s*)?(0x[0-9a-f]+)$", text)
    return int(m.group(4), 16) if m else None


def blocks(ins):
    addr = [a for a, _ in ins]
    pos = {a: i for i, a in enumerate(addr)}
    recs = [i for i, (_, t) in enumerate(ins) if "LDG.E.128.CONSTANT" in t]
    if not recs:
        sys.exit("no colour-record loads (LDG.E.128.CONSTANT) in the kernel")
    loops = []   # (head index, back-edge index)
    fwd = []     # (branch index, target index)
    for i, (a, t) in enumerate(ins):
        tg = branch_target(t)
        if tg is None or tg not in pos:
            continue
        (loops if tg <= a else fwd).append((i, pos[tg]) if tg > a else (pos[tg], i))
    # march loop: the innermost loop around every record load
    around = [(h, e) for h, e in loops if h <= recs[0] and recs[-1] <= e]
    if not around:
        sys.exit("no loop around the record loads")
    lh, le = min(around, key=lambda he: he[1] - he[0])
    # fetch loop: a loop nested in the march loop that does not hold the record loads
    inner = [(h, e) for h, e in loops if lh < h and e < le and not (h <= recs[0] <= e)]
    if not inner:
        sys.exit("no fetch loop inside the march loop")
    fh, fe = max(inner, key=lambda he: sum("LDG" in ins[k][1] for k in range(he[0], he[1] + 1)))
    # shading block: the widest forward branch of the march loop that skips every record load but not the fetch loop
    sk = [(b, t) for b, t in fwd if lh <= b and t <= le and b < recs[0] and recs[-1] < t and b > fe]
    if not sk:
        sys.exit("no branch around the shading block")
    sb, st = max(sk, key=lambda bt: bt[1] - bt[0])
    s0, s1 = sb + 1, st - 1
    # division slow paths inside the shading block: predicated forward branches over a CALL
    slow = set()
    for b, t in fwd:
        body = [ins[k][1] for k in range(b + 1, t)]
        if s0 <= b and t <= s1 + 1 and len(body) <= 8 and any(x.startswith("CALL") for x in body):
            slow.update(range(b + 1, t))
    # fetch-loop exit block: between the fetch loop's back-edge and the target of the branch that skips the loop
    skip = [t for b, t in fwd if lh <= b < fh and fe < t <= s0]
    exit_n = (min(skip) - fe - 1) if skip else 0
    loop_n = le - lh + 1
    fetch_n = fe - fh + 1
    shade_n = s1 - s0 + 1
    return {
        "loop": loop_n,
        "fetch": fetch_n,
        "shade": shade_n,
        "shade_common": shade_n - len(slow),
        "fetch_exit": exit_n,
        "body": loop_n - fetch_n - shade_n - exit_n,
        "ranges": {"loop": (addr[lh], addr[le]), "fetch": (addr[fh], addr[fe]), "shade": (addr[s0], addr[s1])},
    }


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--src", default=ROOT, help="repository root to compile (default: this tree)")
    ap.add_argument("--kbd", default="16,25", help="basis sizes (comma separated)")
    ap.add_argument("--keep", default=None, help="directory that keeps the cubins and SASS listings")
    ap.add_argument("extra", nargs="*", help="more nvcc arguments (after --)")
    a = ap.parse_args()
    out_dir = a.keep or tempfile.mkdtemp(prefix="sass_blocks_")
    os.makedirs(out_dir, exist_ok=True)
    try:
        for kbd in [int(k) for k in a.kbd.split(",")]:
            cubin, log = compile_cubin(os.path.abspath(a.src), kbd, out_dir, a.extra)
            name = next((n for n in kernel_names(kbd) if f"Function properties for {n}" in log), None)
            if name is None:
                sys.exit(f"no batch kernel for KBD={kbd} in {cubin}")
            regs, frame, sst, sld = ptxas_stats(log, name)
            ins = disassemble(cubin, name)
            if a.keep:
                with open(os.path.join(out_dir, f"march_{kbd}.sass"), "w") as f:
                    f.writelines(f"{ad:05x}  {t}\n" for ad, t in ins)
            b = blocks(ins)
            r = b["ranges"]
            print(f"KBD={kbd}  march_persistent_kernel<{kbd}, false, kOutLinear>")
            print(f"  registers {regs}, stack frame {frame} B, spill stores {sst} B, spill loads {sld} B")
            print(f"  march loop  {b['loop']:4d}  [{r['loop'][0]:#x}, {r['loop'][1]:#x}]")
            print(f"  body        {b['body']:4d}  (empty sample, one table fetch)")
            print(f"  fetch loop  {b['fetch']:4d}  [{r['fetch'][0]:#x}, {r['fetch'][1]:#x}]  per extra table fetch"
                  f" (+{b['fetch_exit']} on leaving it)")
            print(f"  shading     {b['shade']:4d}  [{r['shade'][0]:#x}, {r['shade'][1]:#x}]  "
                  f"common path {b['shade_common']} (without the division slow paths)")
            print(f"  lane_sim.c: C_BODY = {b['body']}, C_FETCH = {b['fetch']}, C_SHADE = {b['shade_common']}")
    finally:
        if not a.keep:
            shutil.rmtree(out_dir, ignore_errors=True)


if __name__ == "__main__":
    main()
