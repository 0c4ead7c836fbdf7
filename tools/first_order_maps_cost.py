#!/usr/bin/env python
"""What the voxel-based first-order maps cost: LMInferer.first_order_maps on CUDA tensors and on numpy arrays, the map
kernel alone (lm_first_order_maps_dev), and the numpy statement first_order_maps.maps_host.

    python tools/first_order_maps_cost.py [--out DIR] [--rounds 3]

Builds the engine as bench.py does (R231, the seeded weights of bench.get_weights) and runs, on the int16 phantoms of
oracle.synth (seed 100) at 300 slices of 256x256 and 512x512 with the two-lung mask of tools/statistics_cost.py, the
"lung" row and the lobe row 1, at kernel radius 1, 2 and 3, for all 18 features and for Mean, Variance, Entropy:
  * "device"  LMInferer.first_order_maps on CUDA tensors, CUDA events on the current stream around the call
  * "kernel"  lm_first_order_maps_dev alone with the call's plan, CUDA events around it
  * "numpy"   LMInferer.first_order_maps on numpy arrays, wall time, download of the maps included (radius 1 only)
  * "host"    maps_host, one round, wall time (256x256, radius 1 only)
  * "write_bound_ms"  features x 8 B x voxels at the H100 SXM data sheet's 3.35 TB/s, beside the kernel time
Median over alternating rounds and the spread (max - min).  The card name and power limit come from a read-only
nvidia-smi query.  Writes DIR/first_order_maps_cost.json when --out is given.
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
SUBSET = ("Mean", "Variance", "Entropy")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for first_order_maps_cost.json")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()

    import torch
    import bench
    from statistics_cost import gpu_info, lung_mask
    from lungmask_b200 import LMInferer, first_order_maps as fm
    from oracle import synth

    info = gpu_info()
    print("gpu: %s" % info)
    sd = bench.get_weights(3, bench.WEIGHT_SEEDS[3])
    fd, wpath = tempfile.mkstemp(suffix=".pth", prefix="fom_cost_")
    os.close(fd)
    try:
        torch.save(sd, wpath)
        inferer = LMInferer(modelname="R231", modelpath=wpath, batch_size=20, tqdm_disable=True, device=0)
    finally:
        os.remove(wpath)
    result = {"gpu": info, "workload": "int16 phantom (seed 100), 300-slice two-lung mask", "rounds": args.rounds,
              "unit": "ms", "cases": {}}

    def events(fn):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        e.synchronize()
        return s.elapsed_time(e)

    for hw in (256, 512):
        vol = synth.phantom(SLICES, hw, hw, seed=100)
        mask = lung_mask(SLICES, hw, hw)
        tv, tm = torch.from_numpy(vol).cuda(), torch.from_numpy(mask).cuda()
        for row in ("lung", 1):
            code = 256 if row == "lung" else row
            n_roi = int((mask > 0).sum() if row == "lung" else (mask == row).sum())
            v = vol[mask > 0] if row == "lung" else vol[mask == row]
            plan = fm.plan_maps(n_roi, float(v.min()), float(v.max()), 25, True, 0, n_roi)
            for r in (1, 2, 3):
                table = torch.from_numpy(fm.entropy_table((2 * r + 1) ** 3)).cuda()
                for feats in (None, SUBSET):
                    names = fm.check_features(feats)
                    out = torch.empty((len(names),) + vol.shape, dtype=torch.float64, device="cuda")

                    def kernel():
                        inferer.engine.first_order_maps_dev(
                            tv.data_ptr(), 0, tm.data_ptr(), vol.shape, code, r, True, 25, plan.low, plan.n_levels, True,
                            plan.base, 0, float("nan"), 0.0, fm.feature_bits(names), table.data_ptr(), table.numel(),
                            out.data_ptr(), stream=torch.cuda.current_stream().cuda_stream)

                    def device():
                        inferer.first_order_maps(tv, tm, label=row, features=feats, kernel_radius=r)

                    kernel()   # warm-up: module load
                    device()
                    dev_t, ker_t, np_t = [], [], []
                    for _ in range(args.rounds):
                        ker_t.append(events(kernel))
                        dev_t.append(events(device))
                        if r == 1:
                            t0 = time.perf_counter()
                            inferer.first_order_maps(vol, mask, label=row, features=feats, kernel_radius=r)
                            np_t.append((time.perf_counter() - t0) * 1e3)
                    del out
                    torch.cuda.empty_cache()
                    key = "%dx%d/%s/r%d/%s" % (hw, hw, row, r, "all" if feats is None else "subset")
                    c = {"roi_voxels": n_roi, "maps": len(names),
                         "write_bound_ms": len(names) * 8 * vol.size / 3.35e12 * 1e3}
                    for name, ts in (("device", dev_t), ("kernel", ker_t), ("numpy", np_t)):
                        c[name] = {"median": float(np.median(ts)), "spread": float(np.ptp(ts))} if ts else "not measured"
                    if hw == 256 and r == 1:
                        t0 = time.perf_counter()
                        fm.maps_host(vol, mask, label=row, features=feats, kernel_radius=r)
                        c["host"] = (time.perf_counter() - t0) * 1e3
                    else:
                        c["host"] = "not measured"
                    result["cases"][key] = c
                    print(key, json.dumps(c), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "first_order_maps_cost.json"), "w") as f:
            json.dump(result, f, indent=1)
    inferer.engine.close()


if __name__ == "__main__":
    main()
