#!/usr/bin/env python3
"""A / B timing of two builds of libnfcb200.so on the benchmark's workloads, in one session on one GPU.

Each build is a source tree (its nfc_laboratory_b200/csrc is built with make in a temporary copy) or a prebuilt
libnfcb200.so.  Every build gets its own temporary copy of this tree with its library in place, and bench.py runs from
there, so nothing is written into the trees given.  The builds run alternately --runs times each on the default workload
(nfca106), then once each on every workload of --others.  Per build and workload the script reports phases_ms.ms_lanes,
value and frames_digest of every run, their median and range, and the card's name, power limit and clocks.

usage: python tools/lanes_ab.py A B [--runs 3] [--others nfcb106,nfca424,mixed] [--profile SO] [--out DIR]
  --profile SO   also run the given NFCB200_LANE_PROFILE build once on nfca106 under NFCB200_TRACE=1 and keep its lane
                 profile table (may be given more than once)
  --out DIR      write the JSON lines and the report there as well (default: print only)
"""
import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join("nfc_laboratory_b200", "libnfcb200.so")
BENCH = ["--gpus", "1", "--steps", "5", "--warmup", "2", "--no-e2e", "--no-cpu"]


def tree_copy(dst):
    """what bench.py runs from: itself, the package (without its library), tests/, oracle/, include/ and the peak table"""
    skip = shutil.ignore_patterns("__pycache__", "*.so", "build_ptxas.log")
    os.makedirs(dst)
    for name in ("bench.py", "MEASURED_PEAKS.json"):
        if os.path.exists(os.path.join(ROOT, name)):
            shutil.copy(os.path.join(ROOT, name), dst)
    for name in ("nfc_laboratory_b200", "tests", "oracle", "include"):
        shutil.copytree(os.path.join(ROOT, name), os.path.join(dst, name), symlinks=True, ignore=skip)


def stage(spec, work, label):
    """a runnable copy of this tree whose library is the build `spec` (a source tree or a .so)"""
    dst = os.path.join(work, label)
    tree_copy(dst)
    if spec.endswith(".so"):
        shutil.copy(spec, os.path.join(dst, LIB))
    else:
        src = os.path.join(work, label + "_src")
        shutil.copytree(os.path.join(spec, "nfc_laboratory_b200", "csrc"), os.path.join(src, "nfc_laboratory_b200", "csrc"))
        shutil.copytree(os.path.join(spec, "include"), os.path.join(src, "include"))
        subprocess.check_call(["make", "-s", "-C", os.path.join(src, "nfc_laboratory_b200", "csrc")], stdout=subprocess.DEVNULL)
        shutil.copy(os.path.join(src, LIB), os.path.join(dst, LIB))
    return dst


def card():
    q = "name,power.limit,clocks.max.sm,clocks.max.mem"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))


def bench(tree, workload, env=None):
    p = subprocess.run([sys.executable, os.path.join(tree, "bench.py")] + BENCH + ["--workload", workload], cwd=tree,
                       capture_output=True, text=True, env=env)
    lines = [ln for ln in p.stdout.splitlines() if ln.startswith("{")]
    if p.returncode != 0 or not lines:
        raise SystemExit("bench.py failed in %s (exit %d):\n%s" % (tree, p.returncode, p.stderr[-4000:]))
    return json.loads(lines[-1]), p.stderr


def brief(r):
    return {"ms_lanes": r["phases_ms"]["ms_lanes"], "value": r["value"], "frames_digest": r["frames_digest"],
            "phases_ms": r["phases_ms"], "clocks": r.get("clocks")}


def summary(runs, key):
    v = [r[key] for r in runs]
    return {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("a")
    ap.add_argument("b")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--others", default="nfcb106,nfca424,mixed")
    ap.add_argument("--profile", action="append", default=[])
    ap.add_argument("--out")
    args = ap.parse_args()

    work = tempfile.mkdtemp(prefix="lanes_ab_")
    try:
        trees = {"A": stage(os.path.abspath(args.a), work, "A"), "B": stage(os.path.abspath(args.b), work, "B")}
        info = card()
        print(json.dumps({"card": info, "A": args.a, "B": args.b}), flush=True)
        res = {"A": {}, "B": {}}
        plan = [("nfca106", lab) for _ in range(args.runs) for lab in ("A", "B")]
        plan += [(w, lab) for w in args.others.split(",") if w for lab in ("A", "B")]
        for w, lab in plan:
            r = brief(bench(trees[lab], w)[0])
            res[lab].setdefault(w, []).append(r)
            print(json.dumps(dict(build=lab, workload=w, **r)), flush=True)

        profiles = []
        for k, so in enumerate(args.profile):
            t = stage(os.path.abspath(so), work, "P%d" % k)
            r, err = bench(t, "nfca106", env=dict(os.environ, NFCB200_TRACE="1"))
            table = [ln for ln in err.splitlines() if "lane profile" in ln or ln.startswith("[nfcb200]   ")]
            profiles.append({"so": so, "ms_lanes": r["phases_ms"]["ms_lanes"], "table": table[-9:] if table else []})  # the last call's table: header, 7 classes, total
            print("\n".join(["profile %s" % so] + profiles[-1]["table"]), flush=True)

        report = {"card": info, "builds": {"A": args.a, "B": args.b}, "profiles": profiles, "workloads": {}}
        for w in res["A"]:
            report["workloads"][w] = {lab: {"ms_lanes": summary(res[lab][w], "ms_lanes"), "value": summary(res[lab][w], "value"),
                                            "frames_digest": sorted({r["frames_digest"] for r in res[lab][w]})} for lab in ("A", "B")}
        print("\n%s, power limit %s, max SM clock %s, max memory clock %s" % (info.get("name"), info.get("power.limit"),
                                                                         info.get("clocks.max.sm"), info.get("clocks.max.mem")))
        print("%-8s %5s %28s %28s %s" % ("workload", "build", "ms_lanes median (range)", "value GS/s median (range)", "frames_digest"))
        for w, d in report["workloads"].items():
            for lab in ("A", "B"):
                m, v = d[lab]["ms_lanes"], d[lab]["value"]
                print("%-8s %5s %10.1f (%7.1f - %7.1f) %10.3f (%6.3f - %6.3f) %s" % (w, lab, m["median"], m["min"], m["max"], v["median"] / 1e3,
                                                                                    v["min"] / 1e3, v["max"] / 1e3, ",".join(d[lab]["frames_digest"])))
            same = d["A"]["frames_digest"] == d["B"]["frames_digest"] and len(d["A"]["frames_digest"]) == 1
            print("%-8s frames_digest %s, ms_lanes B / A = %.3f" % (w, "identical" if same else "DIFFERS", d["B"]["ms_lanes"]["median"] / d["A"]["ms_lanes"]["median"]))
        if args.out:
            os.makedirs(args.out, exist_ok=True)
            with open(os.path.join(args.out, "lanes_ab.json"), "w") as f:
                json.dump({"report": report, "runs": res}, f, indent=1)
    finally:
        shutil.rmtree(work, ignore_errors=True)


if __name__ == "__main__":
    main()
