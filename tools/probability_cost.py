#!/usr/bin/env python
"""What the class probabilities cost: LMInferer.apply against LMInferer.apply_with_probabilities.

    python tools/probability_cost.py [--out DIR] [--rounds 3]

Builds the engine as bench.py does (R231, the seeded weights of bench.get_weights, waves of 33 slices) and alternates
the two calls in one process on two 300-slice phantoms (seed 100): 256x256 (the C2 volume) and 512x512.  After one
warm-up call of each, every round runs apply then apply_with_probabilities on each phantom.  Reports, per call, the
per-stage device times of lm_last_timings (CUDA events on the engine stream) and the end-to-end wall time of the Python
call (host copies included), as the median over the rounds and the spread (max - min).  The card name and power
limit come from a read-only nvidia-smi query.  Writes DIR/probability_cost.json when --out is given.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

STAGES = ["h2d", "preprocess", "forward", "postprocess", "reshape", "d2h", "total"]
SLICES = 300


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or r.stderr.strip()
    except Exception as ex:   # the numbers stay valid without it; say why it is missing
        return "nvidia-smi unavailable: %s" % ex


def one_call(inferer, vol, with_probs):
    t0 = time.perf_counter()
    if with_probs:
        mask, probs = inferer.apply_with_probabilities(vol)
    else:
        mask, probs = inferer.apply(vol), None
    wall = (time.perf_counter() - t0) * 1e3
    t = inferer.engine.last_timings()
    row = {k: t[k] for k in STAGES}
    row["wall"] = wall
    return row, mask, probs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for probability_cost.json")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()

    import torch
    import bench
    from lungmask_b200 import LMInferer
    from oracle import synth

    info = gpu_info()
    print("gpu: %s" % info)
    sd = bench.get_weights(3, bench.WEIGHT_SEEDS[3])
    fd, wpath = tempfile.mkstemp(suffix=".pth", prefix="probability_cost_")
    os.close(fd)
    try:
        torch.save(sd, wpath)
        inferer = LMInferer(modelname="R231", modelpath=wpath, batch_size=20, tqdm_disable=True, device=0)
    finally:
        os.remove(wpath)
    vols = {"300x256x256": synth.phantom(SLICES, seed=100), "300x512x512": synth.phantom(SLICES, 512, 512, seed=100)}
    calls = [("apply", False), ("apply_with_probabilities", True)]
    for name, vol in vols.items():                      # warm-up: buffers, graphs
        for _, wp in calls:
            _, mask, _ = one_call(inferer, vol, wp)
    rows = {(v, c): [] for v in vols for c, _ in calls}
    for _ in range(args.rounds):
        for name, vol in vols.items():
            masks = []
            for c, wp in calls:
                row, mask, _ = one_call(inferer, vol, wp)
                rows[(name, c)].append(row)
                masks.append(mask)
            assert np.array_equal(masks[0], masks[1]), "apply_with_probabilities returned another mask than apply"

    result = {"gpu": info, "workload": "R231 (3 classes), bench.get_weights, 300-slice phantoms seed 100, waves of %d"
              % inferer.wave_slices, "rounds": args.rounds, "unit": "ms", "volumes": {}}
    cols = STAGES + ["wall"]
    print("\nms per volume, median of %d rounds (spread max - min)" % args.rounds)
    print("%-12s %-25s " % ("volume", "call") + " ".join("%15s" % c for c in cols))
    for name in vols:
        result["volumes"][name] = {}
        med = {}
        for c, _ in calls:
            r = rows[(name, c)]
            med[c] = {k: float(np.median([x[k] for x in r])) for k in cols}
            spread = {k: float(np.max([x[k] for x in r]) - np.min([x[k] for x in r])) for k in cols}
            result["volumes"][name][c] = {"median": med[c], "spread": spread, "rounds": r}
            print("%-12s %-25s " % (name, c) + " ".join("%8.2f (%4.2f)" % (med[c][k], spread[k]) for k in cols))
        extra = {k: med["apply_with_probabilities"][k] - med["apply"][k] for k in cols}
        result["volumes"][name]["extra"] = extra
        print("%-12s %-25s " % (name, "extra") + " ".join("%15.2f" % extra[k] for k in cols))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "probability_cost.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
