"""Alternated bench.py runs of two builds of the library (A/B: DESIGN.md 7c), per kernel class and end to end.

    python tools/c8_teams_bench.py --a sketchedit_b200/libA.so --b sketchedit_b200/libB.so --runs 5 --out DIR [-- bench.py args]

Runs `bench.py --classes-out` as a subprocess `--runs` times per build, A B A B ..., each with SE_B200_LIB naming the
build. Prints the card's name and power limit, then per build the median and range of `value`, of the batch-1 latencies
and of every kernel class's us / step (one instrumented pass per run). With --dump the first run of each build also
writes its outputs (bench.py --dump-outputs) and the files are compared byte for byte. Nothing else: no clock or power
settings, no profiler.
"""
import argparse
import filecmp
import json
import os
import re
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run_bench(lib, extra, classes_path, dump_dir):
    env = dict(os.environ, SE_B200_LIB=os.path.abspath(lib))
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--classes-out", classes_path] + extra
    if dump_dir:
        cmd += ["--dump-outputs", dump_dir]
    out = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, text=True, check=True).stdout
    line = json.loads([ln for ln in out.splitlines() if ln.startswith("{")][-1])
    classes = {}
    with open(classes_path) as f:
        for ln in f:
            m = re.match(r"\| ([\d.]+) \| [\d.]+ \| `(.+?)` \|", ln)   # class names contain '|'
            if m:
                classes[m.group(2)] = float(m.group(1))
    return line, classes


def med_range(xs):
    return "%.1f [%.1f-%.1f]" % (statistics.median(xs), min(xs), max(xs))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--a", required=True)
    ap.add_argument("--b", required=True)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", required=True)
    ap.add_argument("--dump", action="store_true")
    ap.add_argument("bench_args", nargs="*")
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, text=True).stdout.strip(), flush=True)
    res = {"a": [], "b": []}
    for r in range(args.runs):
        for k in ("a", "b"):
            dump = os.path.join(args.out, "dump_" + k) if args.dump and r == 0 else None
            line, classes = run_bench(getattr(args, k), args.bench_args, os.path.join(args.out, "classes_%s%d.md" % (k, r)), dump)
            res[k].append((line, classes))
            print("run %d %s: value %.1f, %.3f ms/step, clocks %s, latency %s" % (
                r, k, line["value"], line["ms_per_step"], json.dumps(line.get("clocks")), json.dumps(line.get("latency"))), flush=True)
    if args.dump:
        da, db = os.path.join(args.out, "dump_a"), os.path.join(args.out, "dump_b")
        for name in sorted(os.listdir(da)):
            same = filecmp.cmp(os.path.join(da, name), os.path.join(db, name), shallow=False)
            print("outputs %s: %s" % (name, "byte-identical" if same else "DIFFER"))
            os.remove(os.path.join(da, name))
            os.remove(os.path.join(db, name))
    for k in ("a", "b"):
        print("%s = %s: value %s images/s" % (k, getattr(args, k), med_range([l["value"] for l, _ in res[k]])))
    names = sorted(res["a"][0][1], key=lambda n: -res["a"][0][1][n])
    print("| class | a: us / step | b: us / step | b / a |\n|---|---:|---:|---:|")
    for n in names:
        xa = [c[n] for _, c in res["a"] if n in c]
        xb = [c[n] for _, c in res["b"] if n in c]
        if xa and xb:
            print("| %s | %s | %s | %.3f |" % (n, med_range(xa), med_range(xb), statistics.median(xb) / statistics.median(xa)))
    with open(os.path.join(args.out, "result.json"), "w") as f:
        json.dump({k: [{"line": l, "classes": c} for l, c in v] for k, v in res.items()}, f)


if __name__ == "__main__":
    main()
