#!/usr/bin/env python
"""What the first-order features cost: LMInferer.first_order on CUDA tensors and on numpy arrays, and the same features
with the host numpy statement.

    python tools/first_order_cost.py [--out DIR] [--rounds 3]

Builds the engine as bench.py does (R231, the seeded weights of bench.get_weights) and runs, on two 300-slice phantoms
(seed 100) at 256x256 and 512x512, each as int16 (exact rows) and as float32 (the int16 values plus a uniform fraction
in [0, 1): float rows), with the two-lung mask of tools/statistics_cost.py (rows 1, 2 and "lung") and its five-lobe
split of tools/shape_cost.py (rows 1..5 and "lung"), bin width 25.  Per case:
  * "device"  LMInferer.first_order on CUDA tensors (uploaded once), CUDA events on the current stream around the call;
              it ends with a synchronisation, so this is its whole span on the device timeline
  * "numpy"   LMInferer.first_order on the numpy arrays, wall time (the uploads included)
  * "host"    one round of the host statement: numpy statistics and percentiles, first_order.sums_host and the features
              per row
Median over the rounds and the spread (max - min).  The exact rows are checked bit for bit against the host rows.  The
card name and power limit come from a read-only nvidia-smi query.  Writes DIR/first_order_cost.json when --out is given.
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

SLICES = 300
SPACING = (0.703125, 0.703125, 1.25)   # (x, y, z) mm
BIN_WIDTH = 25


def host_rows(vol, mask):
    """{row: FirstOrderRow} of the host statement for the present labels and "lung"."""
    from lungmask_b200 import first_order as fo
    out = {}
    for r in [int(x) for x in np.unique(mask) if x] + [256]:
        v = vol[(mask > 0) if r == 256 else (mask == r)]
        x = v.astype(np.float64)
        plan = fo.plan_row(v.size, float(x.min()), float(x.max()), float(np.mean(x)), np.percentile(x, fo.PERCENTILES),
                           BIN_WIDTH, v.dtype.kind in "iub")
        out[r] = fo.build_row(r, "", BIN_WIDTH, plan, *fo.sums_host(v, plan, BIN_WIDTH), spacing=SPACING)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for first_order_cost.json")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()

    import torch
    import bench
    from shape_cost import lobes_of
    from statistics_cost import gpu_info, lung_mask
    from lungmask_b200 import LMInferer
    from oracle import synth

    info = gpu_info()
    print("gpu: %s" % info)
    sd = bench.get_weights(3, bench.WEIGHT_SEEDS[3])
    fd, wpath = tempfile.mkstemp(suffix=".pth", prefix="first_order_cost_")
    os.close(fd)
    try:
        torch.save(sd, wpath)
        inferer = LMInferer(modelname="R231", modelpath=wpath, batch_size=20, tqdm_disable=True, device=0)
    finally:
        os.remove(wpath)
    rng = np.random.default_rng(100)
    result = {"gpu": info, "workload": "300-slice phantoms seed 100, two-lung and five-lobe masks, bin width 25",
              "rounds": args.rounds, "unit": "ms", "cases": {}}
    print("\n%-34s %14s %16s %10s" % ("case", "device ms", "numpy-input ms", "host ms"))
    for H in (256, 512):
        base = synth.phantom(SLICES, H, H, seed=100)
        lungs = lung_mask(SLICES, H, H)
        for dt in ("int16", "float32"):
            vol = base if dt == "int16" else (base + rng.random(base.shape, dtype=np.float32)).astype(np.float32)
            for masks, mask in (("lungs", lungs), ("lobes", lobes_of(lungs))):
                name = "%dx%dx%d %s %s" % (SLICES, H, H, dt, masks)
                tv, tm = torch.from_numpy(vol).to("cuda:0"), torch.from_numpy(mask).to("cuda:0")
                inferer.first_order(tv, tm, spacing=SPACING)     # warm-up: work buffers, module load
                t0 = time.perf_counter()
                want = host_rows(vol, mask)
                host = (time.perf_counter() - t0) * 1e3
                dev, npy = [], []
                for _ in range(args.rounds):
                    e0, e1 = (torch.cuda.Event(enable_timing=True) for _ in range(2))
                    e0.record()
                    r_dev = inferer.first_order(tv, tm, spacing=SPACING)
                    e1.record()
                    e1.synchronize()
                    dev.append(e0.elapsed_time(e1))
                    t0 = time.perf_counter()
                    r_np = inferer.first_order(vol, mask, spacing=SPACING)
                    npy.append((time.perf_counter() - t0) * 1e3)
                    for r, w in want.items():
                        for got in (r_dev, r_np):
                            g = got["lung" if r == 256 else r]
                            assert np.array_equal(g.histogram, w.histogram), (name, r)
                            if w.exact:
                                assert g.features == w.features and g.power_sums == w.power_sums, (name, r)
                med = {"device": float(np.median(dev)), "numpy": float(np.median(npy)), "host": host}
                spread = {"device": float(np.max(dev) - np.min(dev)), "numpy": float(np.max(npy) - np.min(npy))}
                result["cases"][name] = {"median": med, "spread": spread, "rounds": {"device": dev, "numpy": npy}}
                print("%-34s %7.2f (%5.2f) %8.1f (%5.1f) %10.0f" % (name, med["device"], spread["device"], med["numpy"],
                                                                   spread["numpy"], host), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "first_order_cost.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
