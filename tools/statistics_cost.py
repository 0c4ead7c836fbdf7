#!/usr/bin/env python
"""What the per-label statistics cost: LMInferer.statistics on CUDA tensors and on numpy arrays, against numpy on the host.

    python tools/statistics_cost.py [--out DIR] [--rounds 3]

Builds the engine as bench.py does (R231, the seeded weights of bench.get_weights) and runs, on two 300-slice phantoms
(seed 100) at 256x256 and 512x512, each as int16 and as float32 (the int16 values plus a uniform fraction in [0, 1)),
with an R231-style mask (two ellipsoidal lungs, labels 1 = right and 2 = left, about 30 % of the voxels):
  * "device"  LMInferer.statistics on CUDA tensors (uploaded once), timed with CUDA events on the current stream around
              the call; the call ends with the engine's synchronisation, so this is its whole span on the device timeline
  * "numpy"   LMInferer.statistics on the numpy arrays, wall time (uploads included)
  * "host"    the same numbers with numpy on the host: vol[mask == l] for both labels and the union, mean, std, min, max,
              np.percentile(v, 15) and (v < -950).mean(), wall time
Perc15 and LAA-950, median over the rounds and the spread (max - min).  The achieved bandwidth of the device call counts
(passes over the volume) x (element + 1 mask byte) per voxel against the H100 SXM data-sheet 3.35 TB/s; the passes are
the count and histogram passes, the moments pass of a float volume and the radix-select passes (from the kernel count).
The device results are checked against the host ones (percentiles and counts exactly).  The card name and power limit
come from a read-only nvidia-smi query.  Writes DIR/statistics_cost.json when --out is given.
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

SLICES = 300
HBM_TBS = 3.35


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or r.stderr.strip()
    except Exception as ex:   # the numbers stay valid without it; say why it is missing
        return "nvidia-smi unavailable: %s" % ex


def lung_mask(S, H, W):
    z, y, x = np.ogrid[:S, :H, :W]
    m = np.zeros((S, H, W), np.uint8)
    for label, cx in ((1, 0.32), (2, 0.68)):   # image left = patient right
        m[((z - S / 2) / (0.45 * S)) ** 2 + ((y - 0.5 * H) / (0.3 * H)) ** 2 + ((x - cx * W) / (0.15 * W)) ** 2 <= 1.0] = label
    return m


def host_numbers(vol, mask):
    out = {}
    v64 = vol.astype(np.float64)
    for row in (1, 2, "lung"):
        v = v64[mask > 0] if row == "lung" else v64[mask == row]
        out[row] = (v.size, v.mean(), v.std(), v.min(), v.max(), np.percentile(v, 15), (v < -950).mean())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for statistics_cost.json")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()

    import torch
    import bench
    from lungmask_b200 import LMInferer
    from oracle import synth

    info = gpu_info()
    print("gpu: %s" % info)
    sd = bench.get_weights(3, bench.WEIGHT_SEEDS[3])
    fd, wpath = tempfile.mkstemp(suffix=".pth", prefix="statistics_cost_")
    os.close(fd)
    try:
        torch.save(sd, wpath)
        inferer = LMInferer(modelname="R231", modelpath=wpath, batch_size=20, tqdm_disable=True, device=0)
    finally:
        os.remove(wpath)
    rng = np.random.default_rng(100)
    cases = {}
    for H in (256, 512):
        base = synth.phantom(SLICES, H, H, seed=100)
        mask = lung_mask(SLICES, H, H)
        for dt in ("int16", "float32"):
            vol = base if dt == "int16" else (base + rng.random(base.shape, dtype=np.float32)).astype(np.float32)
            cases["%dx%dx%d %s" % (SLICES, H, H, dt)] = (vol, mask)
    result = {"gpu": info, "workload": "300-slice phantoms seed 100, two-lung ellipsoid mask, Perc15 and LAA-950",
              "rounds": args.rounds, "unit": "ms", "cases": {}}
    print("\n%-22s %16s %8s %8s %16s %16s %10s" % ("case", "device ms", "passes", "GB/s", "numpy-input ms", "host numpy ms",
                                                  "lung %"))
    for name, (vol, mask) in cases.items():
        tv, tm = torch.from_numpy(vol).to("cuda:0"), torch.from_numpy(mask).to("cuda:0")
        torch.cuda.synchronize()
        inferer.statistics(tv, tm)     # warm-up: work buffers, module load
        inferer.statistics(vol, mask)
        dev, npy, host = [], [], []
        for _ in range(args.rounds):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            s_dev = inferer.statistics(tv, tm)
            e1.record()
            e1.synchronize()
            dev.append(e0.elapsed_time(e1))
            launches = inferer.engine.last_timings()["kernel_launches"]
            t0 = time.perf_counter()
            s_np = inferer.statistics(vol, mask)
            npy.append((time.perf_counter() - t0) * 1e3)
            t0 = time.perf_counter()
            want = host_numbers(vol, mask)
            host.append((time.perf_counter() - t0) * 1e3)
            for row, w in want.items():
                for s in (s_dev, s_np):
                    r = s[row]
                    assert r.voxels == w[0] and r.percentile_hu[15.0] == w[5] and r.fraction_below[-950] == w[6], (name, row)
                    assert r.min_hu == w[3] and r.max_hu == w[4], (name, row)
                    assert abs(r.mean_hu - w[1]) <= 1e-12 * abs(w[1]) and abs(r.std_hu - w[2]) <= 1e-12 * w[2], (name, row)
        is_float = vol.dtype.kind == "f"
        select_passes = (launches - 2 - int(is_float)) // 2
        passes = 2 + int(is_float) + select_passes
        nbytes = passes * (vol.dtype.itemsize + 1) * vol.size
        med = {k: float(np.median(v)) for k, v in (("device", dev), ("numpy", npy), ("host", host))}
        spread = {k: float(np.max(v) - np.min(v)) for k, v in (("device", dev), ("numpy", npy), ("host", host))}
        gbs = nbytes / (med["device"] * 1e-3) / 1e9
        result["cases"][name] = {"median": med, "spread": spread, "kernel_launches": launches, "passes": passes,
                                 "bytes": nbytes, "device_GBps": gbs, "share_of_3.35TBps": gbs / (HBM_TBS * 1e3),
                                 "lung_fraction": float((mask > 0).mean()), "rounds": {"device": dev, "numpy": npy, "host": host}}
        print("%-22s %8.2f (%5.2f) %8d %8.0f %8.1f (%5.1f) %8.1f (%5.1f) %10.1f" % (
            name, med["device"], spread["device"], passes, gbs, med["numpy"], spread["numpy"], med["host"], spread["host"],
            100 * (mask > 0).mean()))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "statistics_cost.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
