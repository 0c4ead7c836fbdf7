#!/usr/bin/env python
"""What the wavelet decompositions and their features cost: lm_wavelet_dev per band, and LMInferer.wavelet_features on
CUDA tensors and on numpy arrays.

    python tools/wavelet_cost.py [--out DIR] [--rounds 3]

Builds the engine as bench.py does (R231, the seeded weights of bench.get_weights) and runs, on the int16 300-slice
phantoms (seed 100) at 256x256 and 512x512, with the two-lung mask of tools/statistics_cost.py (rows 1, 2 and "lung")
and its five-lobe split of tools/shape_cost.py (rows 1..5 and "lung"), coif1, bin width 25 and all six feature classes.
Per case, in rounds that alternate the three measurements:
  * "band"    one lm_wavelet_dev call (Engine.wavelet_dev) into a preallocated float64 CUDA tensor: CUDA events on the
              current stream around the 8 bands, divided by 8; every call ends with a synchronisation
  * "device"  wavelet_features on CUDA tensors (uploaded once), CUDA events around the whole call: 16 bands, the
              discretisation check, the first-order and texture calls of all 8 decompositions
  * "numpy"   wavelet_features on the numpy arrays, wall time (the uploads included)
Median over the rounds and the spread (max - min).  The card name and power limit come from a read-only nvidia-smi
query.  Writes DIR/wavelet_cost.json when --out is given.
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
    ap.add_argument("--out", default=None, help="directory for wavelet_cost.json")
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
    fd, wpath = tempfile.mkstemp(suffix=".pth", prefix="wavelet_cost_")
    os.close(fd)
    try:
        torch.save(sd, wpath)
        inferer = LMInferer(modelname="R231", modelpath=wpath, batch_size=20, tqdm_disable=True, device=0)
    finally:
        os.remove(wpath)
    result = {"gpu": info, "workload": "int16 300-slice phantoms seed 100, two-lung and five-lobe masks, coif1, bin width "
              "25, all six classes", "rounds": args.rounds, "unit": "ms", "cases": {}}
    print("\n%-28s %14s %16s %18s" % ("case", "band ms", "device ms", "numpy-input ms"))
    for H in (256, 512):
        vol = synth.phantom(SLICES, H, H, seed=100)
        lungs = lung_mask(SLICES, H, H)
        tv = torch.from_numpy(vol).to("cuda:0")
        band = torch.empty(vol.shape, dtype=torch.float64, device="cuda:0")
        stream = torch.cuda.current_stream().cuda_stream
        for masks, mask in (("lungs", lungs), ("lobes", lobes_of(lungs))):
            name = "%dx%dx%d int16 %s" % (SLICES, H, H, masks)
            tm = torch.from_numpy(mask).to("cuda:0")
            inferer.wavelet_features(tv, tm, bin_width=BIN_WIDTH, spacing=SPACING)   # warm-up: work buffers, module load
            one, dev, npy = [], [], []
            for _ in range(args.rounds):
                e0, e1 = (torch.cuda.Event(enable_timing=True) for _ in range(2))
                e0.record()
                for b in range(8):
                    inferer.engine.wavelet_dev(tv.data_ptr(), _native.DTYPE_I16, vol.shape, "coif1", b, band.data_ptr(),
                                               stream=stream)
                e1.record()
                e1.synchronize()
                one.append(e0.elapsed_time(e1) / 8)
                e0.record()
                inferer.wavelet_features(tv, tm, bin_width=BIN_WIDTH, spacing=SPACING)
                e1.record()
                e1.synchronize()
                dev.append(e0.elapsed_time(e1))
                t0 = time.perf_counter()
                inferer.wavelet_features(vol, mask, bin_width=BIN_WIDTH, spacing=SPACING)
                npy.append((time.perf_counter() - t0) * 1e3)
            med = {"band": float(np.median(one)), "device": float(np.median(dev)), "numpy": float(np.median(npy))}
            spread = {k: float(np.max(v) - np.min(v)) for k, v in (("band", one), ("device", dev), ("numpy", npy))}
            result["cases"][name] = {"median": med, "spread": spread, "rounds": {"band": one, "device": dev, "numpy": npy}}
            print("%-28s %7.3f (%5.3f) %8.1f (%5.1f) %9.1f (%5.1f)" % (name, med["band"], spread["band"], med["device"],
                                                                       spread["device"], med["numpy"], spread["numpy"]),
                  flush=True)
        del band, tv
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "wavelet_cost.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
