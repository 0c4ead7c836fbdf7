#!/usr/bin/env python
"""What the LoG image type and its features cost: one image per call (lm_laplacian_of_gaussian_dev), and
LMInferer.log_features on CUDA tensors and on numpy arrays, against the traffic bound of the nine line passes.

    python tools/log_cost.py [--out DIR] [--rounds 3]

Builds the engine as bench.py does (R231, the seeded weights of bench.get_weights) and runs, on the int16 300-slice
phantoms (seed 100) at 256x256 and 512x512 with spacing (0.703125, 0.703125, 1.25) mm:
  * "sigma=S"  one LoG image at S = 1, 3 and 5 mm into a preallocated float64 CUDA tensor with preallocated work
               volumes: CUDA events on the current stream around the call (which ends with a synchronisation)
  * "bound"    the least time the HBM traffic of one image allows at 3.35 TB/s (the H100 SXM data sheet): 9 passes of
               at least 16 B per voxel (read 8, write 8) plus the 8 B reads of the running sum by the y and z terms,
               160 B per voxel
  * "moved"    the bytes the kernels move per image as designed, over the same bandwidth: each pass reads its input in
               both sweeps, writes and reads back the causal sweep and writes its result (the int16 input is 2 B)
and, with the two-lung mask of tools/statistics_cost.py and its five-lobe split of tools/shape_cost.py, sigma 1, 3 and
5 mm, bin width 25 and all six feature classes:
  * "device"   log_features on CUDA tensors (uploaded once), CUDA events around the whole call
  * "numpy"    log_features on the numpy arrays, wall time (the uploads included)
Rounds alternate the measurements; median over the rounds and the spread (max - min).  The card name and power limit
come from a read-only nvidia-smi query in the same run.  Writes DIR/log_cost.json when --out is given.
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
SIGMAS = (1.0, 3.0, 5.0)
BIN_WIDTH = 25
HBM_BYTES_PER_S = 3.35e12
BOUND_BYTES_PER_VOXEL = 9 * 16 + 2 * 8


def moved_bytes_per_voxel(in_bytes):
    """The bytes per voxel one image moves as the kernels are written: per term, the first pass reads the input twice
    and writes, reads and writes float64 (2 in + 24), the second pass 2 x 8 + 24, the last pass the same plus the
    read of the running sum in the y and z terms."""
    first, other = 2 * in_bytes + 24, 2 * 8 + 24
    return 3 * (first + 2 * other) + 2 * 8


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for log_cost.json")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()

    import torch
    import bench
    from shape_cost import lobes_of
    from statistics_cost import gpu_info, lung_mask
    from lungmask_b200 import LMInferer, _native
    from oracle import synth

    info = gpu_info()
    print("gpu: %s" % info)
    sd = bench.get_weights(3, bench.WEIGHT_SEEDS[3])
    fd, wpath = tempfile.mkstemp(suffix=".pth", prefix="log_cost_")
    os.close(fd)
    try:
        torch.save(sd, wpath)
        inferer = LMInferer(modelname="R231", modelpath=wpath, batch_size=20, tqdm_disable=True, device=0)
    finally:
        os.remove(wpath)
    result = {"gpu": info, "workload": "int16 300-slice phantoms seed 100, spacing %s mm; images at sigma %s mm; "
              "features with the two-lung and five-lobe masks, sigma %s mm, bin width 25, all six classes"
              % (SPACING, SIGMAS, SIGMAS), "rounds": args.rounds, "unit": "ms",
              "bound_bytes_per_voxel": BOUND_BYTES_PER_VOXEL, "moved_bytes_per_voxel": moved_bytes_per_voxel(2),
              "cases": {}}
    image_kinds = ["sigma=%g" % s for s in SIGMAS]
    eng = inferer.engine
    for H in (256, 512):
        vol = synth.phantom(SLICES, H, H, seed=100)
        lungs = lung_mask(SLICES, H, H)
        tv = torch.from_numpy(vol).to("cuda:0")
        out = torch.empty(vol.shape, dtype=torch.float64, device="cuda:0")
        work = [torch.empty(vol.shape, dtype=torch.float64, device="cuda:0") for _ in range(2)]
        stream = torch.cuda.current_stream().cuda_stream

        def one(sigma):
            eng.laplacian_of_gaussian_dev(tv.data_ptr(), _native.DTYPE_I16, vol.shape, SPACING, sigma,
                                          [w.data_ptr() for w in work], out.data_ptr(), stream=stream)

        name = "%dx%dx%d int16 image" % (SLICES, H, H)
        for s in SIGMAS:   # warm-up: modules, the flag
            one(s)
        times = {k: [] for k in image_kinds}
        for _ in range(args.rounds):
            for s, k in zip(SIGMAS, image_kinds):
                e0, e1 = (torch.cuda.Event(enable_timing=True) for _ in range(2))
                e0.record()
                one(s)
                e1.record()
                e1.synchronize()
                times[k].append(e0.elapsed_time(e1))
        med = {k: float(np.median(v)) for k, v in times.items()}
        spread = {k: float(np.max(v) - np.min(v)) for k, v in times.items()}
        med["bound"] = vol.size * BOUND_BYTES_PER_VOXEL / HBM_BYTES_PER_S * 1e3
        med["moved"] = vol.size * moved_bytes_per_voxel(2) / HBM_BYTES_PER_S * 1e3
        result["cases"][name] = {"median": med, "spread": spread, "rounds": times}
        print("%-30s " % name + " ".join("%s %.3f (%.3f)" % (k, med[k], spread[k]) for k in image_kinds) +
              "  bound %.3f  moved %.3f" % (med["bound"], med["moved"]), flush=True)
        del out, work
        for masks, mask in (("lungs", lungs), ("lobes", lobes_of(lungs))):
            name = "%dx%dx%d int16 %s" % (SLICES, H, H, masks)
            tm = torch.from_numpy(mask).to("cuda:0")
            inferer.log_features(tv, tm, SIGMAS, bin_width=BIN_WIDTH, spacing=SPACING)   # warm-up
            times = {"device": [], "numpy": []}
            for _ in range(args.rounds):
                e0, e1 = (torch.cuda.Event(enable_timing=True) for _ in range(2))
                e0.record()
                inferer.log_features(tv, tm, SIGMAS, bin_width=BIN_WIDTH, spacing=SPACING)
                e1.record()
                e1.synchronize()
                times["device"].append(e0.elapsed_time(e1))
                t0 = time.perf_counter()
                inferer.log_features(vol, mask, SIGMAS, bin_width=BIN_WIDTH, spacing=SPACING)
                times["numpy"].append((time.perf_counter() - t0) * 1e3)
            med = {k: float(np.median(v)) for k, v in times.items()}
            spread = {k: float(np.max(v) - np.min(v)) for k, v in times.items()}
            result["cases"][name] = {"median": med, "spread": spread, "rounds": times}
            print("%-30s device %.0f (%.0f)  numpy %.0f (%.0f)" % (name, med["device"], spread["device"], med["numpy"],
                                                                    spread["numpy"]), flush=True)
        del tv
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "log_cost.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
