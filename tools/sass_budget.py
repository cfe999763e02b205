"""Instruction budget of one 16-entry group of the blend backward, counted in its sm_90a SASS.

    python tools/sass_budget.py                 # compiles lara_b200/csrc/render_bwd.cu to a temporary cubin
    python tools/sass_budget.py FILE.cubin      # or an existing cubin
    python tools/sass_budget.py FILE.sass       # or the text of `cuobjdump -sass`

Prints the static instruction counts of the parts of render_bwd_kernel<kEpiFloat> (the default epilogue; the
deterministic instantiations in the same cubin are not counted):

  walk step        the warp's step of 128 list positions outside its chunks: mask loads, compaction into the queue,
                   the carry of a partial chunk (the outermost of the three loops around the groups)
  record gather    the chunk's point_list and record loads into the warp's ring, per 32 entries
  chunk set-up     the rest of the chunk loop before its first group: mask transpose and phase-2 schedule

  phase-1 trip     the per-pixel pair loop (from its head to its back-branch), without the exact re-evaluation of
                   eval_pair_bwd (the smallest forward branch in the loop that jumps over every CALL of it: the IEEE
                   divisions' slow paths), i.e. the fast path of one trip
  between phases   from the phase-1 back-branch to the head of the phase-2 loop: the per-group schedule and set-up
  phase-2 trip     the phase-2 pixel loop, head to back-branch (both branches of the body: ray-splat and low-pass)
  partial sums     from the phase-2 back-branch to the last RED (red.global.add.v4.f32) of the kernel

The ranges are found by their anchors -- the phase-1 loop (the first loop whose body has a MUFU.EX2: the pair's
exp), the loops' back-branches and the REDs -- not by addresses, so the script keeps working when the code moves.
Counts are static (instructions in the range), not dynamic issue counts.

    python tools/sass_budget.py --fwd [FILE]    # the blend forward: lara_b200/csrc/render_fwd.cu

counts render_fwd_kernel<true> (the training instantiation, with the contribution record) by the same kind of anchors:

  staging             from the batch's __syncthreads_count (BAR.RED.POPC) to the barrier after staging (BAR.SYNC):
                      the gathers, the shared stores and, since the cull moved there, the per-tile octagon test
  cull, per 32 slots  the warp's compaction loop after that barrier (the loop with a VOTE.ANY), per ballot: its body
                      over the ballots ptxas unrolled into it
  batch set-up        the rest up to the pixel-mask loop (s_out clearing, loop control)
  phase A, per chunk  the pixel-mask loop (the loop with an F2I: the mask's row bounds), head to back-branch
  trip: loop head     the pair loop (the first loop after phase A whose body has a MUFU.EX2) from its head to its
                      first LDS.U8 (the hit's list entry)
  trip: body          from there to the back-branch: a contributing trip's fast path
  chunk advance       the spans of the pair loop that a trip inside a chunk branches over and that hold a shared store
                      (the write-back of a finished chunk's blended bits): once per 32 hits
  exact paths         the spans that hold a CALL or a double-precision instruction (the IEEE divisions' slow paths and
                      mapped_depth's DP sequence, which runs only where the fp32 estimate cannot settle the rounding)
  record, per batch   from the pair loop's back-branch to the batch loop's back-branch: the saturation exit, the
                      transposes back, the scatter into s_out and the stores
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
SOURCE = "render_bwd.cu"
INSTANTIATION = "ILi0E"   # the default epilogue, kEpiFloat

_INSN = re.compile(r"^\s*/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;")
_F64 = re.compile(r"\bD(?:FMA|MUL|ADD)\b|F64|RCP64H")
_BRA = re.compile(r"\bBRA\b(?:\s+!?U?P\d,)?\s+0x([0-9a-f]+)")


def sass_of(path: str | None) -> str:
    if path and path.endswith(".sass"):
        with open(path) as f:
            return f.read()
    with tempfile.TemporaryDirectory() as tmp:
        cubin = path
        if cubin is None:
            cubin = os.path.join(tmp, "kernel.cubin")
            csrc = os.path.join(ROOT, "lara_b200", "csrc")
            subprocess.run([os.path.join(CUDA, "bin", "nvcc"), "-gencode", "arch=compute_90a,code=sm_90a", "-O3",
                            "-std=c++17", "-I", csrc, "-I", os.path.join(ROOT, "include"), "-cubin", "-o", cubin,
                            os.path.join(csrc, SOURCE)], check=True)
        return subprocess.run([os.path.join(CUDA, "bin", "cuobjdump"), "-sass", cubin], check=True,
                              capture_output=True, text=True).stdout


def kernel_insns(sass: str) -> list[tuple[int, str]]:
    """(address, text) of every instruction of the default-epilogue render_bwd_kernel.

    The cubin holds one instantiation of the kernel per epilogue (render_bwd_kernel<kEpi>); each starts its addresses
    at 0, so only one of them may be read.  The one counted is kEpiFloat (= 0), the path every non-deterministic
    backward runs: its mangled name carries the template argument as ILi0E."""
    out, inside = [], False
    for line in sass.splitlines():
        if "Function :" in line:
            inside = KERNEL + INSTANTIATION in line
            continue
        if inside:
            m = _INSN.match(line)
            if m:
                out.append((int(m.group(1), 16), m.group(2)))
    if not out:
        raise SystemExit(f"no {KERNEL} {INSTANTIATION} in the SASS")
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

    # phase 1: the first loop, by its back-branch, with a MUFU.EX2 in its body
    h1 = b1 = -1
    for i, (a, t) in enumerate(insns):
        m = _BRA.search(t)
        if m and int(m.group(1), 16) <= a:
            head = idx[int(m.group(1), 16)]
            if any("MUFU.EX2" in insns[k][1] for k in range(head, i)):
                h1, b1 = head, i
                break
    if h1 < 0:
        raise SystemExit("phase-1 loop not found")
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
    # the partial sums' REDs (not the REDUX of the warp reductions): the run of them right after phase 2; ptxas may
    # place copies of the group body for divergent warps after the kernel's end, which are not counted
    reds = [i for i, (_, t) in enumerate(insns)
            if t.lstrip("@!P0123456789 ").startswith("RED") and not t.lstrip("@!P0123456789 ").startswith("REDUX")]
    last_red = next(r for r in reds if r > b2)
    while any(last_red < r <= last_red + 8 for r in reds):
        last_red = next(r for r in reds if last_red < r <= last_red + 8)
    # the three loops around the groups, by their back-branches to before phase 1: the 16-entry groups of a chunk,
    # the 32-entry chunks of a walk step, then the warp's walk steps of 128 list positions
    outer = []
    for i in range(last_red, len(insns)):
        m = _BRA.search(insns[i][1])
        if m and int(m.group(1), 16) < insns[h1][0]:
            outer.append((idx[int(m.group(1), 16)], i))
    (gh, gb), (ch, cb), (sh, sb) = outer[0], outer[1], outer[2]
    # the chunk's record gather: from the chunk loop's head to its last 16-byte shared store before the groups (none
    # where the records are staged per step, for the whole CTA)
    gather = max((i for i in range(ch, gh) if "STS.128" in insns[i][1]), default=ch - 1) - ch + 1
    return {
        "walk step (per 128 positions)": (sb - sh + 1) - (cb - ch + 1),
        "record gather (per 32 entries)": gather,
        "chunk set-up (per 32 entries)": gh - ch - gather,
        "group head (to the phase-1 loop)": h1 - gh,
        "phase-1 trip (fast path)": (b1 - h1 + 1) - exact,
        "phase-1 exact re-evaluation": exact,
        "between phases": h2 - (b1 + 1),
        "phase-2 trip": b2 - h2 + 1,
        "partial sums": last_red - b2,
        "group tail (after the REDs)": gb - last_red,
        "REDs": sum(1 for r in reds if b2 < r <= last_red),
    }


def _is_back(insn: tuple[int, str]) -> int | None:
    m = _BRA.search(insn[1])
    return int(m.group(1), 16) if m and int(m.group(1), 16) <= insn[0] else None


def fwd_budget(insns: list[tuple[int, str]]) -> dict[str, int]:
    addr = [a for a, _ in insns]
    idx = {a: i for i, a in enumerate(addr)}

    def loop_with(anchor: str, i0: int) -> tuple[int, int]:
        """(head, back-branch) of the first loop after index i0 whose body holds `anchor`."""
        for i in range(i0, len(insns)):
            t = _is_back(insns[i])
            if t is not None and idx[t] >= i0 and any(anchor in insns[k][1] for k in range(idx[t], i)):
                return idx[t], i
        raise SystemExit(f"no loop with {anchor} after {i0}")

    def spans(h: int, b: int, inner: list[int]) -> set[int]:
        """Indices inside the smallest forward branch of [h, b] that jumps over each index of `inner`."""
        out: set[int] = set()
        for k in inner:
            best = None
            for i in range(h, k):
                m = _BRA.search(insns[i][1])
                if m and int(m.group(1), 16) > insns[i][0]:
                    tgt = idx[int(m.group(1), 16)]
                    if tgt > k and tgt <= b and (best is None or tgt - i < best[1] - best[0]):
                        best = (i, tgt)
            if best:
                out.update(range(best[0] + 1, best[1]))
        return out

    bh = next(i for i, (_, t) in enumerate(insns) if "BAR.RED.POPC" in t)
    bs = next(i for i in range(bh, len(insns)) if "BAR.SYNC" in insns[i][1])
    mh, mb = loop_with("F2I", bs)
    ch, cb = loop_with("VOTE.ANY", bs)
    ballots = sum(1 for k in range(ch, cb) if "VOTE.ANY" in insns[k][1])
    ph, pb = loop_with("MUFU.EX2", mb)
    exact = spans(ph, pb, [i for i in range(ph, pb) if "CALL" in insns[i][1] or _F64.search(insns[i][1])])
    advance = spans(ph, pb, [i for i in range(ph, pb) if insns[i][1].lstrip("@!P0123456789 ").startswith("STS")]) - exact
    lu8 = next(i for i in range(ph, pb) if "LDS.U8" in insns[i][1])
    rare = exact | advance
    batch_end = next(i for i in range(pb + 1, len(insns)) if (t := _is_back(insns[i])) is not None and idx[t] <= bh)
    return {
        "staging (per batch)": bs - bh + 1,
        "cull, per 32 slots": round((cb - ch + 1) / max(ballots, 1)),
        "batch set-up (rest, to phase A)": (mh - bs - 1) - (cb - ch + 1),
        "phase A, per chunk": mb - mh + 1,
        "trip: loop head": sum(1 for i in range(ph, lu8) if i not in rare),
        "trip: body (fast path)": sum(1 for i in range(lu8, pb + 1) if i not in rare),
        "chunk advance (per 32 hits)": len(advance),
        "exact paths": len(exact),
        "record (per batch)": batch_end - pb,
    }


def main() -> None:
    args = sys.argv[1:]
    fwd = "--fwd" in args
    args = [a for a in args if a != "--fwd"]
    path = args[0] if args else None
    if fwd:
        global KERNEL, SOURCE, INSTANTIATION
        KERNEL, SOURCE, INSTANTIATION = "render_fwd_kernel", "render_fwd.cu", "ILb1E"
    res = fwd_budget(kernel_insns(sass_of(path))) if fwd else budget(kernel_insns(sass_of(path)))
    for k, v in res.items():
        print(f"{k:34s} {v:5d}")


if __name__ == "__main__":
    main()
