"""Instruction budget of one 16-entry group of the blend backward, counted in its sm_90a SASS.

    python tools/sass_budget.py                 # compiles lara_b200/csrc/render_bwd.cu to a temporary cubin
    python tools/sass_budget.py FILE.cubin      # or an existing cubin
    python tools/sass_budget.py FILE.sass       # or the text of `cuobjdump -sass`

Prints the static instruction counts of the four parts of render_bwd_kernel that a group runs through:

  phase-1 trip     the per-pixel pair loop (from its head to its back-branch), without the exact re-evaluation of
                   eval_pair_bwd (the smallest forward branch in the loop that jumps over every CALL of it: the IEEE
                   divisions' slow paths), i.e. the fast path of one trip
  between phases   from the phase-1 back-branch to the head of the phase-2 loop: the per-group schedule and set-up
  phase-2 trip     the phase-2 pixel loop, head to back-branch (both branches of the body: ray-splat and low-pass)
  partial sums     from the phase-2 back-branch to the last RED (red.global.add.v4.f32) of the kernel

The ranges are found by their anchors -- the REDUX.MAX that starts phase 1 (the warp's trip count), the loops'
back-branches and the REDs -- not by addresses, so the script keeps working when the code moves.  Counts are static
(instructions in the range), not dynamic issue counts.
"""
from __future__ import annotations

import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")
KERNEL = "render_bwd_kernel"

_INSN = re.compile(r"^\s*/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;")
_BRA = re.compile(r"\bBRA\b(?:\s+!?U?P\d,)?\s+0x([0-9a-f]+)")


def sass_of(path: str | None) -> str:
    if path and path.endswith(".sass"):
        with open(path) as f:
            return f.read()
    with tempfile.TemporaryDirectory() as tmp:
        cubin = path
        if cubin is None:
            cubin = os.path.join(tmp, "render_bwd.cubin")
            csrc = os.path.join(ROOT, "lara_b200", "csrc")
            subprocess.run([os.path.join(CUDA, "bin", "nvcc"), "-gencode", "arch=compute_90a,code=sm_90a", "-O3",
                            "-std=c++17", "-I", csrc, "-I", os.path.join(ROOT, "include"), "-cubin", "-o", cubin,
                            os.path.join(csrc, "render_bwd.cu")], check=True)
        return subprocess.run([os.path.join(CUDA, "bin", "cuobjdump"), "-sass", cubin], check=True,
                              capture_output=True, text=True).stdout


def kernel_insns(sass: str) -> list[tuple[int, str]]:
    """(address, text) of every instruction of render_bwd_kernel."""
    out, inside = [], False
    for line in sass.splitlines():
        if "Function :" in line:
            inside = KERNEL in line
            continue
        if inside:
            m = _INSN.match(line)
            if m:
                out.append((int(m.group(1), 16), m.group(2)))
    if not out:
        raise SystemExit(f"no {KERNEL} in the SASS")
    return out


def budget(insns: list[tuple[int, str]]) -> dict[str, int]:
    addr = [a for a, _ in insns]
    idx = {a: i for i, a in enumerate(addr)}

    def back_branch_after(i0: int) -> tuple[int, int]:
        """(head index, branch index) of the first loop whose back-branch follows index i0."""
        for i in range(i0, len(insns)):
            m = _BRA.search(insns[i][1])
            if m and int(m.group(1), 16) <= insns[i][0]:
                tgt = idx[int(m.group(1), 16)]
                if tgt >= i0:
                    return tgt, i
        raise SystemExit("loop not found")

    redux = next(i for i, (_, t) in enumerate(insns) if "REDUX.MAX" in t)
    h1, b1 = back_branch_after(redux)
    # the exact re-evaluation: the smallest forward branch of the loop that skips every CALL in it
    calls = [i for i in range(h1, b1 + 1) if "CALL" in insns[i][1]]
    exact = 0
    if calls:
        spans = []
        for i in range(h1, b1 + 1):
            m = _BRA.search(insns[i][1])
            if m and int(m.group(1), 16) > insns[i][0]:
                tgt = idx[int(m.group(1), 16)]
                if i < calls[0] and tgt > calls[-1]:
                    spans.append(tgt - i - 1)
        exact = min(spans) if spans else 0
    h2, b2 = back_branch_after(b1 + 1)
    reds = [i for i, (_, t) in enumerate(insns) if t.lstrip("@!P0123456789 ").startswith("RED")]
    last_red = max(r for r in reds if r > b2)
    # the two loops around the groups, by their back-branches to before phase 1: the 16-entry groups of a chunk,
    # then the 32-entry chunks of a batch
    outer = []
    for i in range(last_red, len(insns)):
        m = _BRA.search(insns[i][1])
        if m and int(m.group(1), 16) < insns[redux][0]:
            outer.append((idx[int(m.group(1), 16)], i))
    (gh, gb), (ch, _) = outer[0], outer[1]
    return {
        "chunk set-up (per 32 entries)": gh - ch,
        "group head (to REDUX.MAX)": redux - gh + 1,
        "phase-1 trip (fast path)": (b1 - h1 + 1) - exact,
        "phase-1 exact re-evaluation": exact,
        "between phases": h2 - (b1 + 1),
        "phase-2 trip": b2 - h2 + 1,
        "partial sums": last_red - b2,
        "group tail (after the REDs)": gb - last_red,
        "REDs": sum(1 for r in reds if r > b2),
    }


def main() -> None:
    path = sys.argv[1] if len(sys.argv) > 1 else None
    for k, v in budget(kernel_insns(sass_of(path))).items():
        print(f"{k:30s} {v:5d}")


if __name__ == "__main__":
    main()
