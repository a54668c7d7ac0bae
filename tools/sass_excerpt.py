#!/usr/bin/env python
"""SASS listings of the hot kernels (the instruction-mix arguments of DESIGN.md can be checked against these).

    python tools/sass_excerpt.py mash_b200/libmashgpu.so OUT_DIR

writes, per kernel, `<name>.sass` (its innermost loops as cuobjdump prints them, encodings stripped, plus every TMA / mbarrier
instruction) and `summary.md` with the opcode histogram, the static share of the pipes and the opcode mix of each innermost loop."""
import collections
import os
import re
import subprocess
import sys

KERNELS = {
    "scan_kernel_k21_canonical_ascii": "_ZN7mashgpu11scan_kernelILi21ELb1ELb0ELb0EEEvNS_8ScanArgsE",
    "scan_kernel_k21_canonical_packed": "_ZN7mashgpu11scan_kernelILi21ELb1ELb1ELb0EEEvNS_8ScanArgsE",
    "scan_kernel_k21_canonical_ascii_screen": "_ZN7mashgpu11scan_kernelILi21ELb1ELb0ELb1EEEvNS_8ScanArgsE",
    "scan_bytes_kernel_k9": "_ZN7mashgpu17scan_bytes_kernelILi9EEEvNS_8ScanArgsE",        # protein sketches and the translated screen
    "translate6_kernel": "_ZN7mashgpu17translate6_kernelEPKhmiiPhNS_8TrFramesE",
    "dist_kernel": "_ZN7mashgpu11dist_kernelENS_8DistArgsE",
    "dist_probe_kernel": "_ZN7mashgpu17dist_probe_kernelENS_8DistArgsE",
    "dist_pair_kernel": "_ZN7mashgpu16dist_pair_kernelENS_8DistArgs",
    "within_kernel": "_ZN7mashgpu13within_kernelENS_10WithinArgsE",
    "within_pair_kernel": "_ZN7mashgpu18within_pair_kernelENS_10WithinArgsE",
}
PIPES = {
    "ALU (SHF/LOP3/IADD3/PRMT/ISETP/SEL/...)": ("SHF", "LOP3", "IADD3", "IADD", "PRMT", "ISETP", "SEL", "LEA", "MOV", "PLOP3", "HSETP2", "VOTE", "POPC", "FLO", "BREV", "IABS", "IMNMX", "VIMNMX", "LOP"),
    "FMA-pipe integer (IMAD*)": ("IMAD",),
    "LSU shared (LDS/STS/ATOMS)": ("LDS", "STS", "ATOMS", "LDSM"),
    "LSU global (LDG/STG/ATOMG/RED)": ("LDG", "STG", "ATOMG", "RED", "ATOM", "LD", "ST"),
    "control (BRA/BSSY/BSYNC/...)": ("BRA", "BSSY", "BSYNC", "EXIT", "CALL", "RET", "WARPSYNC", "BAR", "NOP", "YIELD"),
    "TMA / bulk copy (UTMALDG/UBLKCP)": ("UTMALDG", "UBLKCP", "UTMASTG"),
    "tensor (HMMA/UTCMMA/...)": ("HMMA", "IMMA", "UTCHMMA", "UTCIMMA", "UTCQMMA"),
}


def opcode(t):
    return re.sub(r"^@!?U?P\w+\s+", "", t).split()[0].split(".")[0]


def hot_path_line(body):
    """The scan kernel's hot path: its longest innermost loop minus the blocks that the branch after each warp vote
    (VOTE.ANY) skips when no lane has a survivor -- i.e. what a warp issues per 8 windows when nobody passes the filter.
    The filter-word kernels have no vote in the loop (pass masks are resolved after it), so there it is the whole loop; the
    control instructions it holds are listed."""
    skip = []
    for i, (_, t) in enumerate(body):
        if t.startswith("VOTE.ANY"):
            for j in range(i + 1, min(i + 6, len(body))):
                m = re.search(r"@!?P\d BRA.*?0x([0-9a-f]+)", body[j][1])
                if m:
                    skip.append((body[j][0] + 1, int(m.group(1), 16)))
                    break
    hot = [(a, t) for a, t in body if not any(x <= a < y for x, y in skip)]
    c = collections.Counter(opcode(t) for _, t in hot)
    alu = sum(n for o, n in c.items() if o in PIPES["ALU (SHF/LOP3/IADD3/PRMT/ISETP/SEL/...)"] + ("VIADD",))
    ctl = ", ".join(f"{o} {c[o]}" for o in ("VOTE", "CALL", "BSSY", "BSYNC", "BRA") if c[o]) or "none"
    what = f"without the {len(skip)} survivor blocks behind the warp votes" if skip else "no warp vote in it: the whole loop"
    span = body[-1][0] + 16 - body[0][0]
    return (f"hot path (longest innermost loop, {what}): {len(hot)} "
            f"instructions per lane per loop trip, {span} bytes of code; ALU pipe {alu}, IMAD {c['IMAD']}, STL {c['STL']}, LDL {c['LDL']}, S2R {c['S2R']}; "
            f"control: {ctl}")


def main():
    so, out = sys.argv[1], sys.argv[2]
    os.makedirs(out, exist_ok=True)
    dump = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True, check=True).stdout.splitlines()
    starts = {i: l.split("Function : ")[1].strip() for i, l in enumerate(dump) if "Function : " in l}
    idx = sorted(starts)
    summary = ["# SASS of the hot kernels (sm_90a), from `cuobjdump -sass mash_b200/libmashgpu.so` via tools/sass_excerpt.py", ""]
    for name, mangled in KERNELS.items():
        at = [i for i in idx if starts[i].startswith(mangled)]
        if not at:
            summary.append(f"## {name}: not found in {so}\n")
            continue
        a = at[0]
        b = idx[idx.index(a) + 1] if idx.index(a) + 1 < len(idx) else len(dump)
        ins = []
        for l in dump[a:b]:
            m = re.match(r"\s+/\*([0-9a-f]{4,})\*/\s+(.*?);", l)
            if m:
                ins.append((int(m.group(1), 16), m.group(2).strip()))
        excerpt = [f"// {mangled}: {len(ins)} instructions; the innermost loops, longest first (full listing: cuobjdump -sass)"]
        ops = collections.Counter()
        for _, t in ins:
            t2 = re.sub(r"^@!?U?P\d+\s+", "", t)
            ops[t2.split()[0].split(".")[0]] += 1
        total = sum(ops.values())
        summary.append(f"## {name}  (`{mangled}`): {total} instructions")
        summary.append("")
        summary.append("| pipe / class | static instructions | share |")
        summary.append("|---|---|---|")
        for pipe, names in PIPES.items():
            n = sum(c for o, c in ops.items() if o in names)
            summary.append(f"| {pipe} | {n} | {100.0 * n / max(1, total):.1f} % |")
        summary.append("")
        summary.append("opcode histogram: " + ", ".join(f"{o} {c}" for o, c in ops.most_common(24)))
        # innermost loops (backward branches whose body holds no other backward branch), longest first
        loops = []
        for addr, t in ins:
            m2 = re.search(r"BRA.*?0x([0-9a-f]+)", t)
            if not m2:
                continue
            tgt = int(m2.group(1), 16)
            if tgt >= addr:
                continue
            body = [x for x in ins if tgt <= x[0] <= addr]
            inner = True
            for y in body[:-1]:
                m3 = re.search(r"BRA.*?0x([0-9a-f]+)", y[1])
                if m3 and int(m3.group(1), 16) < y[0]:
                    inner = False
                    break
            if inner:
                loops.append(body)
        loops.sort(key=len, reverse=True)
        if name.startswith("scan_kernel") and loops:
            summary.append("")
            summary.append(hot_path_line(loops[0]))
        for body in loops[:8]:
            lo = collections.Counter(re.sub(r"^@!?U?P\d+\s+", "", t).split()[0].split(".")[0] for _, t in body)
            summary.append("")
            summary.append(f"innermost loop, {len(body)} instructions ({body[-1][0] + 16 - body[0][0]} bytes) at {body[0][0]:#x}..{body[-1][0]:#x}: " + ", ".join(f"{o} {c}" for o, c in lo.most_common(12)))
        for i, body in enumerate(loops[:4]):
            # the scan kernels' hot loop in full, so that its control flow can be read off the listing
            keep = 1200 if i == 0 and name.startswith("scan_kernel") else 400
            excerpt.append(f"\n// ---- loop {body[0][0]:#x}..{body[-1][0]:#x} ({len(body)} instructions)")
            excerpt += [f"/*{addr:05x}*/  {t}" for addr, t in body[:keep]]
            if len(body) > keep:
                excerpt.append(f"// ... {len(body) - keep} more")
        tma = [f"/*{addr:05x}*/  {t}" for addr, t in ins if re.search(r"UBLKCP|UTMALDG|SYNCS|UTMASTG", t)]
        if tma:
            excerpt.append("\n// ---- TMA / mbarrier instructions in this kernel")
            excerpt += tma[:40]
        open(os.path.join(out, name + ".sass"), "w").write("\n".join(excerpt) + "\n")
        summary.append("")
    open(os.path.join(out, "summary.md"), "w").write("\n".join(summary) + "\n")
    print("\n".join(summary))


if __name__ == "__main__":
    main()
