"""Trimmed SASS evidence: mnemonic histogram per kernel, the TMA / mbarrier instructions, and the hot
loop of march_kernel and of the two hot compositing kernels (cuobjdump -sass on the in-tree .so)."""
import collections
import re
import subprocess
import sys

so = sys.argv[1] if len(sys.argv) > 1 else "nerfacc_b200/csrc/libnerfacc_b200.so"
txt = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
funcs, cur = collections.OrderedDict(), None
for line in txt.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        cur = m.group(1)
        funcs[cur] = []
        continue
    m = re.match(r"\s+/\*([0-9a-f]{4,5})\*/\s+(.*?);", line)
    if m and cur:
        funcs[cur].append((int(m.group(1), 16), m.group(2).strip()))


def demangle(n):
    return subprocess.run(["c++filt", n], capture_output=True, text=True).stdout.strip()


print("# SASS of", so, "(cuobjdump -sass, sm_90a)\n")
for name, ins in funcs.items():
    d = demangle(name)
    if not any(k in d for k in ("march_kernel<true, 16>", "march_kernel<(bool)1, (int)16>", "Cfg<false, true, true>",
                                "expand_samples_kernel", "occ_threshold_pack", "vis_mask_kernel<(bool)0>")):
        continue
    hist = collections.Counter(re.sub(r"^@!?U?P\d+\s+", "", t).split()[0].split(".")[0] for _, t in ins)
    print(f"## {d}\n{len(ins)} instructions; top mnemonics: " + ", ".join(f"{k} {v}" for k, v in hist.most_common(14)))
    tma = [t for _, t in ins if t.split()[0].startswith(("UBLKCP", "SYNCS", "UTMA")) or " UBLKCP" in t or "SYNCS." in t]
    if tma:
        print("TMA / mbarrier: " + "; ".join(sorted(set(re.sub(r"\s+", " ", t) for t in tma))[:8]))
    # hot loop: the innermost backward branch region containing the characteristic instruction
    key = "SHF.R.U64" if "march" in d else "MUFU.EX2"
    idx = [i for i, (_, t) in enumerate(ins) if key in t]
    if idx:
        addr_of = {a: i for i, (a, _) in enumerate(ins)}
        best = None
        for i, (a, t) in enumerate(ins):
            m = re.search(r"BRA(?:\.\w+)*\s+(?:!?U?P\d+,\s*)?0x([0-9a-f]+)", t)
            if m:
                tgt = int(m.group(1), 16)
                if tgt < a and tgt in addr_of and any(addr_of[tgt] <= k <= i for k in idx):
                    span = (addr_of[tgt], i)
                    if best is None or span[1] - span[0] < best[1] - best[0]:
                        best = span
        if best:
            print(f"hot loop: {best[1] - best[0] + 1} instructions")
            for a, t in ins[best[0]:best[1] + 1][:110]:
                print(f"    /*{a:04x}*/ {t}")
    print()
