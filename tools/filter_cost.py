#!/usr/bin/env python
"""What the Square, SquareRoot, Logarithm, Exponential and Gradient image types and their features cost: one image per
call (lm_image_filter_dev / lm_gradient_dev), and LMInferer.filtered_features on CUDA tensors and on numpy arrays.

    python tools/filter_cost.py [--out DIR] [--rounds 3]

Builds the engine as bench.py does (R231, the seeded weights of bench.get_weights) and runs, on the int16 300-slice
phantoms (seed 100) at 256x256 and 512x512, with the two-lung mask of tools/statistics_cost.py (rows 1, 2 and "lung")
and its five-lobe split of tools/shape_cost.py (rows 1..5 and "lung"), all five image types, bin width 25 and all six
feature classes.  Per case, in rounds that alternate the measurements:
  * per image type  one call into a preallocated float64 CUDA tensor (the int16 phantom takes the table path; its
                    table is uploaded once before timing): CUDA events on the current stream; every call ends with a
                    synchronisation
  * "range"         one lm_image_range_dev call
  * "device"        filtered_features on CUDA tensors (uploaded once), CUDA events around the whole call: the range
                    pass, 10 images, the discretisation check, the first-order and texture calls of all 5 images
  * "numpy"         filtered_features on the numpy arrays, wall time (the uploads included)
Median over the rounds and the spread (max - min).  The card name and power limit come from a read-only nvidia-smi
query in the same run.  Writes DIR/filter_cost.json when --out is given.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for filter_cost.json")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()

    import torch
    import bench
    from shape_cost import lobes_of
    from statistics_cost import gpu_info, lung_mask
    from lungmask_b200 import LMInferer, _native
    from lungmask_b200 import filters as flt
    from oracle import synth

    info = gpu_info()
    print("gpu: %s" % info)
    sd = bench.get_weights(3, bench.WEIGHT_SEEDS[3])
    fd, wpath = tempfile.mkstemp(suffix=".pth", prefix="filter_cost_")
    os.close(fd)
    try:
        torch.save(sd, wpath)
        inferer = LMInferer(modelname="R231", modelpath=wpath, batch_size=20, tqdm_disable=True, device=0)
    finally:
        os.remove(wpath)
    result = {"gpu": info, "workload": "int16 300-slice phantoms seed 100, two-lung and five-lobe masks, all five image "
              "types, bin width 25, all six classes", "rounds": args.rounds, "unit": "ms", "cases": {}}
    kinds = list(flt.NAMES) + ["range", "device", "numpy"]
    print("\n%-28s " % "case" + " ".join("%15s" % k for k in kinds))
    eng = inferer.engine
    for H in (256, 512):
        vol = synth.phantom(SLICES, H, H, seed=100)
        lungs = lung_mask(SLICES, H, H)
        tv = torch.from_numpy(vol).to("cuda:0")
        out = torch.empty(vol.shape, dtype=torch.float64, device="cuda:0")
        stream = torch.cuda.current_stream().cuda_stream
        lo, hi = eng.image_range_dev(tv.data_ptr(), _native.DTYPE_I16, vol.shape, stream=stream)
        span = flt.table_span(_native.DTYPE_I16, lo, hi)
        tables = {n: torch.from_numpy(flt.table(n, *span)).to("cuda:0") for n in flt.ELEMENTWISE}

        def one(name):
            if name == "gradient":
                eng.gradient_dev(tv.data_ptr(), _native.DTYPE_I16, vol.shape, SPACING, out.data_ptr(), stream=stream)
            elif name == "range":
                eng.image_range_dev(tv.data_ptr(), _native.DTYPE_I16, vol.shape, stream=stream)
            else:
                eng.image_filter_dev(tv.data_ptr(), _native.DTYPE_I16, vol.shape, name, 0.0, out.data_ptr(),
                                     table=(tables[name].data_ptr(), span[0], span[1]), stream=stream)

        for masks, mask in (("lungs", lungs), ("lobes", lobes_of(lungs))):
            name = "%dx%dx%d int16 %s" % (SLICES, H, H, masks)
            tm = torch.from_numpy(mask).to("cuda:0")
            inferer.filtered_features(tv, tm, bin_width=BIN_WIDTH, spacing=SPACING)   # warm-up: work buffers, modules
            times = {k: [] for k in kinds}
            for _ in range(args.rounds):
                for k in list(flt.NAMES) + ["range"]:
                    e0, e1 = (torch.cuda.Event(enable_timing=True) for _ in range(2))
                    e0.record()
                    one(k)
                    e1.record()
                    e1.synchronize()
                    times[k].append(e0.elapsed_time(e1))
                e0, e1 = (torch.cuda.Event(enable_timing=True) for _ in range(2))
                e0.record()
                inferer.filtered_features(tv, tm, bin_width=BIN_WIDTH, spacing=SPACING)
                e1.record()
                e1.synchronize()
                times["device"].append(e0.elapsed_time(e1))
                t0 = time.perf_counter()
                inferer.filtered_features(vol, mask, bin_width=BIN_WIDTH, spacing=SPACING)
                times["numpy"].append((time.perf_counter() - t0) * 1e3)
            med = {k: float(np.median(v)) for k, v in times.items()}
            spread = {k: float(np.max(v) - np.min(v)) for k, v in times.items()}
            result["cases"][name] = {"median": med, "spread": spread, "rounds": times}
            print("%-28s " % name + " ".join("%8.3f (%4.2f)" % (med[k], spread[k]) if k not in ("device", "numpy")
                                             else "%8.0f (%4.0f)" % (med[k], spread[k]) for k in kinds), flush=True)
        del out, tv, tables
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "filter_cost.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
