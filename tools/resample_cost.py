#!/usr/bin/env python
"""What resampling to 1 mm costs (LMInferer.resample; lm_bspline_coefficients_dev, lm_resample_dev), and what it does to
`texture`.

    python tools/resample_cost.py [--out DIR] [--rounds 3]

Builds the engine as bench.py does (R231, the seeded weights of bench.get_weights) and runs, on the int16 300-slice
phantoms (seed 100) at 256x256 (spacing 1.40625 x 1.40625 x 1.25 mm) and 512x512 (0.703125 x 0.703125 x 1.25 mm, the
same field of view), with the two-lung mask of tools/statistics_cost.py, B-spline resampling to (1, 1, 1) mm.  Per case,
in rounds that alternate the measurements:
  * "decompose"   one lm_bspline_coefficients_dev call into a preallocated float64 CUDA tensor: CUDA events
  * "evaluate"    one lm_resample_dev call (B-spline) from those coefficients and preallocated tables and outputs
  * "device"      LMInferer.resample on CUDA tensors (uploaded once), CUDA events around the whole call
  * "numpy"       LMInferer.resample on the numpy arrays, wall time (the uploads and downloads included)
  * "texture"     LMInferer.texture (GLCM and GLSZM, bin width 25) on the native CUDA pair and on the resampled one
Median over the rounds and the spread (max - min).  Beside the times it prints the least time the data sheet's 3.35 TB/s
of HBM3 bandwidth allows: the decomposition moves (2 + 8) + 16 + 16 bytes per input voxel (the x pass reads int16 and
writes float64; the y and z passes read and write float64), the evaluation reads the coefficients once and writes
2 + 1 bytes per output voxel.  The card name and power limit come from a read-only nvidia-smi query in the same run.
Writes DIR/resample_cost.json when --out is given.
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
TARGET = (1.0, 1.0, 1.0)
HBM_BYTES_PER_MS = 3.35e9   # 3.35 TB/s


def _events():
    import torch
    return [torch.cuda.Event(enable_timing=True) for _ in range(2)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for resample_cost.json")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()

    import torch
    import bench
    from statistics_cost import gpu_info, lung_mask
    from lungmask_b200 import LMInferer, _native
    from lungmask_b200 import resample as rsm
    from oracle import synth

    info = gpu_info()
    print("gpu: %s" % info)
    sd = bench.get_weights(3, bench.WEIGHT_SEEDS[3])
    fd, wpath = tempfile.mkstemp(suffix=".pth", prefix="resample_cost_")
    os.close(fd)
    try:
        torch.save(sd, wpath)
        inferer = LMInferer(modelname="R231", modelpath=wpath, batch_size=20, tqdm_disable=True, device=0)
    finally:
        os.remove(wpath)
    result = {"gpu": info, "workload": "int16 300-slice phantoms seed 100, two-lung mask, B-spline to 1 mm; texture GLCM "
              "and GLSZM at bin width 25", "rounds": args.rounds, "unit": "ms", "cases": {}}
    kinds = ["decompose", "evaluate", "device", "numpy", "texture_native", "texture_resampled"]
    print("\n%-34s " % "case" + " ".join("%17s" % k for k in kinds))
    eng = inferer.engine
    for H, sp in ((256, (1.40625, 1.40625, 1.25)), (512, (0.703125, 0.703125, 1.25))):
        vol = synth.phantom(SLICES, H, H, seed=100)
        mask = lung_mask(SLICES, H, H)
        tv, tm = torch.from_numpy(vol).to("cuda:0"), torch.from_numpy(mask).to("cuda:0")
        g = rsm.grid(vol.shape, sp, TARGET, *rsm.bounding_box(mask))
        coeff = torch.empty(vol.shape, dtype=torch.float64, device="cuda:0")
        tables = [torch.from_numpy(t).to("cuda:0") for t in g.tables[::-1]]
        out = torch.empty(g.shape, dtype=torch.int16, device="cuda:0")
        out_mask = torch.empty(g.shape, dtype=torch.uint8, device="cuda:0")
        stream = torch.cuda.current_stream().cuda_stream
        n_in, n_out = int(np.prod(vol.shape)), int(np.prod(g.shape))
        bound = {"decompose": n_in * (2 + 8 + 16 + 16) / HBM_BYTES_PER_MS, "evaluate": (n_in * 8 + n_out * 3) / HBM_BYTES_PER_MS}

        def decompose():
            eng.bspline_coefficients_dev(tv.data_ptr(), _native.DTYPE_I16, vol.shape, coeff.data_ptr(), stream=stream)

        def evaluate():
            eng.resample_dev(tv.data_ptr(), _native.DTYPE_I16, coeff.data_ptr(), tm.data_ptr(), vol.shape,
                             [t.data_ptr() for t in tables], g.shape, "bspline", out.data_ptr(), out_mask.data_ptr(),
                             stream=stream)

        def device():
            return inferer.resample(tv, tm, TARGET, spacing=sp)

        r = device()   # warm-up: work buffers, modules
        decompose()
        evaluate()
        inferer.texture(tv, tm, spacing=sp)
        inferer.texture(r.image, r.mask, spacing=r.spacing)
        name = "%dx%dx%d int16 -> %dx%dx%d" % ((SLICES, H, H) + g.shape)
        times = {k: [] for k in kinds}
        for _ in range(args.rounds):
            for k, f in (("decompose", decompose), ("evaluate", evaluate), ("device", device),
                         ("texture_native", lambda: inferer.texture(tv, tm, spacing=sp)),
                         ("texture_resampled", lambda: inferer.texture(r.image, r.mask, spacing=r.spacing))):
                e0, e1 = _events()
                e0.record()
                f()
                e1.record()
                e1.synchronize()
                times[k].append(e0.elapsed_time(e1))
            t0 = time.perf_counter()
            inferer.resample(vol, mask, TARGET, spacing=sp)
            times["numpy"].append((time.perf_counter() - t0) * 1e3)
        med = {k: float(np.median(v)) for k, v in times.items()}
        spread = {k: float(np.max(v) - np.min(v)) for k, v in times.items()}
        result["cases"][name] = {"median": med, "spread": spread, "rounds": times, "hbm_bound_ms": bound,
                                 "input_voxels": n_in, "output_voxels": n_out}
        print("%-34s " % name + " ".join("%9.3f (%5.2f)" % (med[k], spread[k]) for k in kinds), flush=True)
        print("%-34s decompose >= %.3f ms, evaluate >= %.3f ms at 3.35 TB/s" % ("", bound["decompose"], bound["evaluate"]),
              flush=True)
        del coeff, out, out_mask, tables, tv, tm, r
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "resample_cost.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
