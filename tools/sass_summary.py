#!/usr/bin/env python3
"""Instruction summary of libnfcb200.so per kernel (cuobjdump -sass, no GPU needed): the mnemonics that prove the Hopper
paths (TMA bulk copy = UBLKCP, mbarrier = SYNCS.*, per-thread async copy = LDGSTS, warp reductions = REDUX / CREDUX, shuffles = SHFL) and the memory mix
(shared LDS / STS vs generic LD / ST vs local LDL / STL).

usage: python tools/sass_summary.py [path to .so] > sass_summary.md
"""
import collections
import re
import subprocess
import sys

so = sys.argv[1] if len(sys.argv) > 1 else "nfc_laboratory_b200/libnfcb200.so"
out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
kern = None
counts = collections.OrderedDict()
for ln in out.splitlines():
    m = re.search(r"Function : (\S+)", ln)
    if m:
        kern = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
        kern = re.sub(r"\((?!anonymous).*", "", kern).replace("nfcb200::", "").replace("(anonymous namespace)::", "")
        counts[kern] = collections.Counter()
        continue
    m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", ln)
    if m and kern:
        op = m.group(1)
        c = counts[kern]
        c["total"] += 1
        for key, pat in (("UBLKCP (cp.async.bulk)", r"^UBLKCP"), ("SYNCS (mbarrier)", r"^SYNCS"), ("LDGSTS (cp.async)", r"^LDGSTS"),
                         ("LDS", r"^LDS"), ("STS", r"^STS"),
                         ("LDG / LD.E (global / generic load)", r"^(LDG|LD\.E|LD$)"), ("STG / ST.E (global / generic store)", r"^(STG|ST\.E|ST$)"),
                         ("LDL", r"^LDL"), ("STL", r"^STL"), ("SHFL", r"^SHFL"), ("REDUX / CREDUX", r"^C?REDUX"), ("MUFU", r"^MUFU"),
                         ("FFMA", r"^FFMA"), ("FADD / FMUL", r"^(FADD|FMUL)"), ("BAR / WARPSYNC", r"^(BAR|WARPSYNC)"), ("ATOM / RED", r"^(ATOM|RED)"),
                         ("HMMA / UTC*MMA (tensor)", r"^(HMMA|UTC.*MMA)")):
            if re.match(pat, op):
                c[key] += 1
print("# SASS instruction summary of `%s` (sm_90a, `cuobjdump -sass`)\n" % so)
print("Static instruction counts per kernel. `UBLKCP` is the TMA bulk copy (`cp.async.bulk`), `SYNCS.*` its mbarrier; no tensor-core")
print("instruction appears anywhere: the path has no dense contraction.  `-fmad=false`: FFMA only where the source asks for it")
print("(`__fmaf_rn` in the screening kernel, the IEEE sqrt / div sequences).\n")
keys = ["total", "UBLKCP (cp.async.bulk)", "SYNCS (mbarrier)", "LDGSTS (cp.async)", "LDS", "STS", "LDG / LD.E (global / generic load)", "STG / ST.E (global / generic store)", "LDL", "STL",
        "SHFL", "REDUX / CREDUX", "MUFU", "FFMA", "FADD / FMUL", "BAR / WARPSYNC", "ATOM / RED", "HMMA / UTC*MMA (tensor)"]
print("| kernel | " + " | ".join(keys) + " |")
print("|---|" + "---:|" * len(keys))
for k, c in counts.items():
    print("| `%s` | " % k + " | ".join(str(c.get(x, 0)) for x in keys) + " |")
