"""A/B of two builds of this library on one GPU: this tree against a base tree (for example the parent commit), in one
process tree, runs interleaved so that clock and neighbour noise fall on both builds alike.

    git archive <base-commit> | tar -x -C <dir>         # any directory git ignores, e.g. build/ab_base
    python scripts/linear_ab_bench.py --base <dir> [--c2-runs 3] [--out <dir>]

Each build runs its own bench.py from its own tree (the base is built with its own recipe if it has no library yet):
  * c2 (`--no-cpu-baseline`) --c2-runs times per build, alternating; each line's `value`, `stage_ms_rank0`,
    `roofline_linear` and `clocks` are printed;
  * c3, c5 and c4 once per build, alternating;
  * outputs: c2, c3 and c5 with `--dump-outputs`, `out.npy` compared bitwise; the c4 parameter gradients with
    torch.use_deterministic_algorithms on (compared bitwise) and off (max abs difference relative to max |base|, against
    the 5e-5 bar of the GEMM tests).
Dumps go to --out (default: a temporary directory).  Prints JSON lines; the last one is the summary.
"""
import argparse
import glob
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = ("metric", "value", "stage_ms_rank0", "roofline_linear", "clocks", "gpu", "gpu_name", "workload")
# c4 under torch.use_deterministic_algorithms(True); warn_only leaves torch's own ops of the benchmark's step running
DET_WRAPPER = ("import runpy, sys, torch; torch.use_deterministic_algorithms(True, warn_only=True); "
               "sys.argv = ['bench.py'] + sys.argv[1:]; runpy.run_path('bench.py', run_name='__main__')")


def ensure_built(tree):
    if not os.path.exists(os.path.join(tree, "pyhgt_b200", "libhgt_b200.so")):
        subprocess.run([sys.executable, "-m", "pyhgt_b200.build"], cwd=tree, check=True)


def run_bench(tree, tag, config, dump=None, det=False, extra=()):
    args = ["--gpus", "1", "--config", config, "--no-cpu-baseline"] + list(extra)
    if dump:
        args += ["--dump-outputs", dump]
    cmd = [sys.executable, "-c", DET_WRAPPER] + args if det else [sys.executable, "bench.py"] + args
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8") if det else None
    r = subprocess.run(cmd, cwd=tree, capture_output=True, text=True, env=env)
    line = None
    for ln in r.stdout.splitlines():
        if ln.startswith("{"):
            try:
                line = json.loads(ln)
            except ValueError:
                pass
    if r.returncode != 0 or line is None:
        print(json.dumps({"build": tag, "config": config, "det": det, "error": r.returncode,
                          "stderr_tail": r.stderr[-2000:]}), flush=True)
        return None
    short = {k: line[k] for k in KEYS if k in line}
    print(json.dumps(dict(build=tag, config=config, det=det, **short)), flush=True)
    return line


def compare(a_dir, b_dir, bitwise):
    """{file: max |b - a| / max(1e-30, max |a|)} over the .npy files of a_dir; bitwise: also whether all are equal."""
    res, equal = {}, True
    for fa in sorted(glob.glob(os.path.join(a_dir, "*.npy"))):
        name = os.path.basename(fa)
        fb = os.path.join(b_dir, name)
        if not os.path.exists(fb):
            res[name] = "missing"
            equal = False
            continue
        a, b = np.load(fa), np.load(fb)
        same = a.shape == b.shape and a.tobytes() == b.tobytes()
        equal &= same
        if a.shape == b.shape:
            res[name] = 0.0 if same else float(np.abs(b.astype(np.float64) - a).max() / max(1e-30, np.abs(a).max()))
        else:
            res[name] = "shape %s vs %s" % (a.shape, b.shape)
    if not res:
        equal = False
    return {"bitwise_equal": equal, "max_rel_diff": max((v for v in res.values() if isinstance(v, float)), default=None),
            "files": len(res)} if bitwise else {"max_rel_diff": max((v for v in res.values() if isinstance(v, float)),
                                                                    default=None), "files": len(res)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", required=True, help="tree of the build to compare against")
    ap.add_argument("--c2-runs", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for the output dumps (default: a temporary one)")
    args = ap.parse_args()
    trees = [("base", os.path.abspath(args.base)), ("this", ROOT)]
    for _, t in trees:
        ensure_built(t)
    out = args.out or tempfile.mkdtemp(prefix="linear_ab_")
    d = lambda tag, name: os.path.join(out, tag, name)                      # noqa: E731
    values = {"base": [], "this": []}
    stages = {"base": [], "this": []}
    for i in range(args.c2_runs):
        for tag, tree in (trees if i % 2 == 0 else trees[::-1]):
            line = run_bench(tree, tag, "c2", dump=d(tag, "c2") if i == 0 else None)
            if line:
                values[tag].append(line["value"])
                stages[tag].append(line.get("stage_ms_rank0"))
    others = {}
    for config in ("c3", "c5", "c4"):
        for tag, tree in trees:
            line = run_bench(tree, tag, config, dump=d(tag, config))
            others.setdefault(config, {})[tag] = line["value"] if line else None
    for tag, tree in trees:
        run_bench(tree, tag, "c4", dump=d(tag, "c4_det"), det=True)
    summary = {"c2_value": values,
               "c2_speedup_median": (float(np.median(values["this"]) / np.median(values["base"]))
                                     if values["this"] and values["base"] else None),
               "c2_ranges_overlap": (min(values["this"]) <= max(values["base"]) and
                                     min(values["base"]) <= max(values["this"])) if values["this"] and values["base"]
               else None,
               "other_value": others,
               "outputs": {c: compare(d("base", c), d("this", c), bitwise=True) for c in ("c2", "c3", "c5", "c4_det")}}
    summary["outputs"]["c4"] = compare(d("base", "c4"), d("this", "c4"), bitwise=False)
    summary["outputs"]["c4"]["within_5e-5"] = (summary["outputs"]["c4"]["max_rel_diff"] is not None and
                                               summary["outputs"]["c4"]["max_rel_diff"] <= 5e-5)
    print(json.dumps({"summary": summary}), flush=True)


if __name__ == "__main__":
    main()
