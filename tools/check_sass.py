#!/usr/bin/env python
"""Static checks of the built library's SASS (cuobjdump works without a GPU) and the evidence file the docs cite:
which kernels use the TMA path (UTMALDG + mbarrier SYNCS), that each ingest LUT gather is one 128-bit + one 64-bit load,
that the strip egress
prefetches into L1 and has no local memory, spill or barrier (it also prints the length of its main loop), and that the Phase egress clips NaN to 1.0 with an explicit select (OpenCV's max(min(v,1),0)) instead
of a .SAT folded into the producing FFMA (round-1 hardware failure).  Usage: python tools/check_sass.py [out.txt]"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "live-video-magnification_b200", "libmagcore_b200.so")


def kernels():
    out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    cur, body = None, collections.OrderedDict()
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip() or m.group(1)
            cur = re.sub(r"mc::\(anonymous namespace\)::", "", cur)
            body[cur] = []
        elif cur and re.match(r"\s+/\*[0-9a-f]{4}\*/", line):
            body[cur].append(re.sub(r"\s*/\*.*?\*/\s*", " ", line).strip())
    return body


def clip_spills(kernel="k_level_clip", source="mc_laplace"):
    """-> {mangled `kernel` instance: (spill store bytes, spill load bytes)} from the build's ptxas -v log of `source`."""
    log = os.path.join(ROOT, "live-video-magnification_b200", "csrc", source + ".ptxas.log")
    out, cur = {}, None
    for line in open(log) if os.path.exists(log) else []:
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur = m.group(1) if kernel in m.group(1) else None
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            out[cur] = (int(m.group(1)), int(m.group(2)))
            cur = None
    return out


def main_loop(lines):
    """-> (first, last) line of a kernel's longest loop: the target of its longest backward branch and that branch
    (cuobjdump prints one 16-byte instruction per line, from offset 0)."""
    best = (0, -1)
    for i, l in enumerate(lines):
        m = re.search(r"\bBRA\b.*?0x([0-9a-f]+)", l)
        if m and int(m.group(1), 16) // 16 < i and i - int(m.group(1), 16) // 16 > best[1] - best[0]:
            best = (int(m.group(1), 16) // 16, i)
    return best


def loop_counts(lines):
    """-> (instructions of the longest loop, those of them that a warp-vote branch skips: the strip egress's dark-end
    spline, which runs only when a lane of the warp needs it)"""
    s, e = main_loop(lines)
    rare = 0
    for i in range(s, e + 1):
        m = re.match(r"VOTE\.ANY (P\d)", lines[i])
        if not m:
            continue
        for j in range(i + 1, e + 1):
            b = re.match(r"@!" + m.group(1) + r" BRA 0x([0-9a-f]+)", lines[j])
            if b:
                rare += max(0, int(b.group(1), 16) // 16 - j - 1)
                break
    return e - s + 1, rare


def main():
    body = kernels()
    count = lambda k, pat: sum(1 for l in body[k] if re.search(pat, l))
    lines, ok = [], True
    lines.append("SASS evidence of libmagcore_b200.so (cuobjdump -sass; tools/check_sass.py)\n")
    lines.append(f"{'kernel':90s} instr  UTMALDG SYNCS LDG.128 LDG.64 CCTL.PF1 SHFL  BAR")
    for k in body:
        lines.append(f"{k[:90]:90s} {len(body[k]):5d}  {count(k, 'UTMALDG'):7d} {count(k, 'SYNCS'):5d} {count(k, r'LDG\.E\.128'):7d} {count(k, r'LDG\.E\.64'):6d} "
                     f"{count(k, r'CCTL\.E\.PF1'):8d} {count(k, 'SHFL'):4d} {count(k, r'BAR\.SYNC'):4d}")

    def need(cond, what):
        nonlocal ok
        lines.append(("ok   " if cond else "FAIL ") + what)
        ok = ok and cond

    lines.append("")
    tma = [k for k in body if k.startswith("void k_level<0, true")]
    need(bool(tma) and all(count(k, "UTMALDG") >= 1 and count(k, "SYNCS") >= 2 for k in tma), "k_level<f32, TMA, *>: cp.async.bulk.tensor (UTMALDG) + mbarrier (SYNCS)")
    pre = [k for k in tma if k.startswith("void k_level<0, true, true")]
    need(bool(pre) and all(count(k, "UTMALDG") == 3 for k in pre), "k_level<f32, TMA, PREFETCH>: three bulk-tensor copies (input window + both state tiles)")
    clip = [k for k in body if k.startswith("void k_level_clip<0, true>")]
    need(len(clip) == 1 and count(clip[0], "UTMALDG") >= 1 and count(clip[0], "SYNCS") >= 2,
         "k_level_clip<f32, TMA>: double-buffered cp.async.bulk.tensor (UTMALDG) + mbarrier (SYNCS)")
    spills = clip_spills()
    need(bool(spills) and all(s == (0, 0) for s in spills.values()), f"k_level_clip<*>: no local-memory spills (ptxas -v, {len(spills)} instances)")
    pclip = [k for k in body if k.startswith("void k_riesz_phase_clip<true>")]
    need(len(pclip) == 1 and count(pclip[0], "UTMALDG") >= 1 and count(pclip[0], "SYNCS") >= 2,
         "k_riesz_phase_clip<TMA>: double-buffered cp.async.bulk.tensor (UTMALDG) + mbarrier (SYNCS)")
    pspills = clip_spills("k_riesz_phase_clip", "mc_riesz")
    need(len(pspills) == 2 and all(s == (0, 0) for s in pspills.values()),
         f"k_riesz_phase_clip<*>: no local-memory spills (ptxas -v, {len(pspills)} instances)")
    r9 = [k for k in body if k.startswith("k_riesz_analysis(") or k.startswith("k_riesz_collapse(")]
    need(len(r9) == 2 and all(count(k, "UTMALDG") == 1 and count(k, "SYNCS") >= 2 for k in r9), "k_riesz_analysis / k_riesz_collapse: 9x9 input tile by one bulk-tensor copy")
    ing = [k for k in body if k.startswith("void k_ingest_lab<")]
    need(bool(ing) and all(count(k, r"LDG\.E\.128") >= 8 and count(k, r"LDG\.E\.128") == count(k, r"LDG\.E\.64") for k in ing),
         "k_ingest_lab: each LUT gather is one LDG.E.128 + one LDG.E.64 (the 24 used bytes of a 32-byte cell)")
    strip = [k for k in body if k.startswith("void k_egress_strip<3")]
    need(bool(strip) and all(count(k, r"CCTL\.E\.PF1") >= 8 and count(k, r"BAR\.SYNC") == 0 for k in strip), "k_egress_strip<3,*>: L1 prefetches, no barrier")
    need(bool(strip) and all(count(k, r"\b(STL|LDL)\b") == 0 for k in strip), "k_egress_strip<3,*>: no local memory (STL / LDL)")
    espills = clip_spills("k_egress_strip")
    need(len(espills) == len(strip) + 2 and all(s == (0, 0) for s in espills.values()),
         f"k_egress_strip<*>: no spills (ptxas -v, {len(espills)} instances)")
    luma = [k for k in strip if k.startswith("void k_egress_strip<3, 1,")]
    need(len(luma) == 4, f"k_egress_strip<3, 1, *>: L-only synthesis at every register cap and with the float tap ({len(luma)} instances)")
    for k in strip:
        n, rare = loop_counts(body[k])
        lines.append(f"     {k}: main loop {n} instructions ({n - rare} outside the warp-voted dark-end spline) "
                     f"per 2 output rows x 4 columns per lane")
    front = [k for k in body if k.startswith("void k_chain_front<")]
    need(len(front) == 3 and all(count(k, r"\b(STL|LDL)\b") == 0 for k in front), "k_chain_front<BGR, gray, NV12>: no local memory (STL / LDL)")
    fspills = clip_spills("k_chain_front", "mc_preprocess")
    need(len(fspills) == 3 and all(s == (0, 0) for s in fspills.values()), f"k_chain_front<*>: no spills (ptxas -v, {len(fspills)} instances)")
    rz = [k for k in body if k.startswith("k_riesz_egress") or "k_riesz_egress(" in k]
    # the select is either an FSEL per channel or a saturate predicated on the NaN test over a preset 1.0
    nan_sel = lambda k: count(k, "FSEL") + count(k, r"@!P\d FADD\.SAT")
    need(bool(rz) and all(count(k, r"FSETP\.NAN") >= 3 and nan_sel(k) >= 3 and count(k, r"FFMA\.SAT") == 0 for k in rz),
         "k_riesz_egress: explicit NaN -> 1.0 select before the gamma (FSETP.NAN + FSEL or @!P FADD.SAT), no FFMA.SAT")
    text = "\n".join(lines) + "\n"
    if len(sys.argv) > 1:
        open(sys.argv[1], "w").write(text)
    print(text)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
