"""Before / after record of a GEMM epilogue change: this checkout against another built checkout (e.g. the parent commit's,
a side-by-side copy that is not part of the repository), alternated in one GPU session so that both see the same card
and clocks.  Per round and build: profiles/gemm_bench.py --graph --backend 3 --epilogue E for every epilogue, then
bench.py --gpus 1 --steps 20 --warmup 3 --no-cpu-baseline --no-extra.  Also: bench.py --dump-outputs of both builds for
every workload, compared file for file.
usage (GPU box): python profiles/epilogue_ab.py --parent DIR --out FILE.json [--rounds 2]
The record goes to FILE.json and the dumped outputs to directories beside it; nothing is written into either checkout."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPILOGUES = ("bias", "residual", "gelu", "dgelu")
WORKLOADS = ("clip_b32", "detr_r50", "lxmert", "clip_l14_336")


def last_json(text):
    for line in reversed(text.splitlines()):
        if line.startswith("{") or line.startswith("["):
            return json.loads(line)
    raise RuntimeError("no JSON line in:\n" + text[-2000:])


def run(cmd, cwd):
    r = subprocess.run(cmd, cwd=cwd, capture_output=True, text=True)
    if r.returncode:
        raise RuntimeError(f"{' '.join(cmd)} (in {cwd}) exited {r.returncode}:\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}")
    return r.stdout


def gemm(tree, epi):
    out = run([sys.executable, os.path.join(HERE, "profiles", "gemm_bench.py"), "--graph", "--backend", "3", "--epilogue", epi,
               "--tree", tree], HERE)
    return {f"{d['M']}x{d['N']}x{d['K']}": d["us"] for d in last_json(out)}


def bench(tree):
    d = last_json(run([sys.executable, "bench.py", "--gpus", "1", "--steps", "20", "--warmup", "3", "--no-cpu-baseline",
                       "--no-extra"], tree))
    return dict(value=d["value"], ms_per_step=d["ms_per_step"], gemm_ms_per_step=d["roofline"]["gemm_ms_per_step"],
                serial_step_ms=d["roofline"]["serial_step_ms"], gemm_tflops=d["roofline"]["achieved"], clocks=d["clocks"])


def same_outputs(trees, out_dir):
    res = {}
    for w in WORKLOADS:
        dirs = []
        for name, tree in trees.items():
            d = os.path.join(out_dir, f"dump_{name}_{w}")
            run([sys.executable, "bench.py", "--gpus", "1", "--steps", "2", "--warmup", "1", "--no-cpu-baseline", "--no-extra",
                 "--workload", w, "--dump-outputs", d], tree)
            dirs.append(d)
        files = sorted(os.listdir(dirs[0]))
        assert files == sorted(os.listdir(dirs[1])), w
        differ = [f for f in files if not np.array_equal(np.load(os.path.join(dirs[0], f)), np.load(os.path.join(dirs[1], f)),
                                                         equal_nan=True)]
        res[w] = dict(files=len(files), differ=differ)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", required=True)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", required=True, help="JSON record; the --dump-outputs directories go beside it")
    args = ap.parse_args()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    trees = {"parent": os.path.abspath(args.parent), "this": HERE}
    smi = run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], HERE).strip()
    rec = dict(gpu=smi, rounds=[])
    for r in range(args.rounds):
        order = list(trees.items()) if r % 2 == 0 else list(trees.items())[::-1]
        rnd = {}
        for name, tree in order:
            rnd[name] = dict(gemm_us={e: gemm(tree, e) for e in EPILOGUES}, bench=bench(tree))
            print(name, json.dumps(rnd[name]), flush=True)
        rec["rounds"].append(rnd)
        with open(args.out, "w") as fh:
            json.dump(rec, fh, indent=1)
    rec["outputs"] = same_outputs(trees, os.path.dirname(os.path.abspath(args.out)))
    print(json.dumps(rec["outputs"]), flush=True)
    with open(args.out, "w") as fh:
        json.dump(rec, fh, indent=1)


if __name__ == "__main__":
    main()
