#!/usr/bin/env python
"""What the GLCM / GLSZM texture features cost: LMInferer.texture on CUDA tensors and on numpy arrays, the lm_glcm_dev
call alone, and the same matrices on the host with numpy / scipy.

    python tools/texture_cost.py [--out DIR] [--rounds 3] [--classes glcm,glszm,glrlm,gldm,ngtdm]

With --classes, the run below is replaced by the one of classes_cost: the GLRLM / GLDM / NGTDM calls alone and the
whole call with those classes against the default one, on the int16 phantoms at both sizes and bin widths.

Builds the engine as bench.py does (R231, the seeded weights of bench.get_weights) and runs, on two 300-slice phantoms
(seed 100) at 256x256 and 512x512, each as int16 and as float32 (the int16 values plus a uniform fraction in [0, 1)),
with the two-lung mask of tools/statistics_cost.py (three rows: both lungs and "lung"), at bin width 25 (about 45
levels: the GLCM counters of every direction in shared memory) and 10 (about 110 levels: the near-diagonal band in
shared memory, the rest in global memory).  Per case:
  * "device"  LMInferer.texture on CUDA tensors (uploaded once), CUDA events on the current stream around the call; it
              ends with a synchronisation, so this is its whole span on the device timeline
  * "glcm"    lm_glcm_dev alone on the "lung" row's level map (Engine.glcm_dev), CUDA events around the call
  * "numpy"   LMInferer.texture on the numpy arrays, wall time (the uploads included)
  * "host"    the same matrices on the host, one round: numpy level maps, slicing + np.bincount for the 13 directions,
              scipy.ndimage.label per level for the zones (the features themselves are host code in both)
Median over the rounds and the spread (max - min).  Every device matrix is checked against the host one.  The card name
and power limit come from a read-only nvidia-smi query.  Writes DIR/texture_cost.json when --out is given.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))   # _texture_ref: the numpy GLRLM / GLDM / NGTDM references

SLICES = 300


def host_rows(vol, mask, bw):
    """{row: (U, zones)} on the host for rows 1, 2 and "lung"."""
    import scipy.ndimage as ndi
    from lungmask_b200 import texture as tx
    out = {}
    for row in (1, 2, "lung"):
        sel = (mask > 0) if row == "lung" else (mask == row)
        vals = vol[sel]
        low, ng = tx.discretisation(float(vals.min()), float(vals.max()), bw)
        L = np.zeros(vol.shape, np.uint8)
        L[sel] = tx.levels(vals, bw, low)
        T = ng * (ng + 1) // 2
        U = np.zeros((13, T), np.int64)
        n = L.shape
        for d, off in enumerate(tx.OFFSETS):
            src = tuple(slice(max(0, -o), n[k] - max(0, o)) for k, o in enumerate(off))
            dst = tuple(slice(max(0, o), n[k] - max(0, -o)) for k, o in enumerate(off))
            a, b = L[src].astype(np.int64), L[dst].astype(np.int64)
            both = (a > 0) & (b > 0)
            i, j = np.minimum(a, b)[both], np.maximum(a, b)[both]
            U[d] = np.bincount((i - 1) * ng - (i - 1) * (i - 2) // 2 + (j - i), minlength=T)
        zones = []
        box = L[ndi.find_objects(sel.astype(np.uint8))[0]]   # the row's bounding box, as PyRadiomics crops to the mask
        for lv in range(1, ng + 1):
            lab, k = ndi.label(box == lv, np.ones((3, 3, 3), bool))
            if k:
                s, c = np.unique(np.bincount(lab.ravel())[1:], return_counts=True)
                zones += [(lv, int(x), int(y)) for x, y in zip(s, c)]
        out[row] = (U, np.array(zones, np.int64).reshape(-1, 3), L, ng)
    return out


def classes_cost(inferer, classes, rounds, info):
    """--classes: on the int16 phantoms, lm_glrlm_dev and lm_neighbour_counts_dev alone on the "lung" row's level map,
    and LMInferer.texture with `classes` and with the default classes, CUDA events around each call.  The "lung" row's
    device matrices (of the calls alone and of the whole call) are checked against the numpy references of
    tests/_texture_ref.py."""
    import torch
    from statistics_cost import lung_mask
    from _texture_ref import glrlm_ref, neighbour_ref
    from lungmask_b200 import texture as tx
    from oracle import synth
    classes = tx.check_classes(classes)
    result = {"gpu": info, "workload": "300-slice int16 phantoms seed 100, two-lung ellipsoid mask, classes %s" % ",".join(classes),
              "rounds": rounds, "unit": "ms", "cases": {}}
    print("\n%-26s %5s %14s %14s %14s %14s" % ("case", "Ng", "glrlm ms", "neighbour ms", "call ms", "default ms"))
    for H in (256, 512):
        vol = synth.phantom(SLICES, H, H, seed=100)
        mask = lung_mask(SLICES, H, H)
        tv, tm = torch.from_numpy(vol).to("cuda:0"), torch.from_numpy(mask).to("cuda:0")
        sel = mask > 0
        for bw in (25, 10):
            name = "%dx%dx%d int16 bw %d" % (SLICES, H, H, bw)
            vals = vol[sel]
            low, ng = tx.discretisation(float(vals.min()), float(vals.max()), bw)
            L = np.zeros(vol.shape, np.uint8)
            L[sel] = tx.levels(vals, bw, low)
            P, (G, N, A) = glrlm_ref(L, ng), neighbour_ref(L, ng, 0)
            tL = torch.from_numpy(L).to("cuda:0")
            st = torch.cuda.current_stream().cuda_stream
            inferer.texture(tv, tm, bin_width=bw, classes=classes)     # warm-up: work buffers, module load
            inferer.texture(tv, tm, bin_width=bw)
            times = {"glrlm": [], "neighbour": [], "call": [], "default": []}
            for _ in range(rounds):
                e = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
                e[0].record()
                runs = inferer.engine.glrlm_dev(tL.data_ptr(), L.shape, ng, stream=st)
                e[1].record()
                nb = inferer.engine.neighbour_counts_dev(tL.data_ptr(), L.shape, ng, 0, stream=st)
                e[2].record()
                res = inferer.texture(tv, tm, bin_width=bw, classes=classes)
                e[3].record()
                inferer.texture(tv, tm, bin_width=bw)
                e[4].record()
                e[4].synchronize()
                for k, (a, b) in zip(times, ((0, 1), (1, 2), (2, 3), (3, 4))):
                    times[k].append(e[a].elapsed_time(e[b]))
                assert np.array_equal(runs, P) and all(np.array_equal(x, y) for x, y in zip(nb, (G, N, A))), name
                r = res["lung"]
                if "glrlm" in classes:
                    assert np.array_equal(r.glrlm_runs, tx.runs_from_counts(P)), name
                if "gldm" in classes:
                    assert np.array_equal(r.gldm_counts, G), name
                if "ngtdm" in classes:
                    assert np.array_equal(r.ngtdm_counts, N) and np.array_equal(r.ngtdm_sums, A), name
            med = {k: float(np.median(v)) for k, v in times.items()}
            spread = {k: float(np.max(v) - np.min(v)) for k, v in times.items()}
            result["cases"][name] = {"median": med, "spread": spread, "n_levels_lung": ng, "rounds": times}
            print("%-26s %5d %7.2f (%5.2f) %7.2f (%5.2f) %7.1f (%5.1f) %7.1f (%5.1f)" % (
                name, ng, med["glrlm"], spread["glrlm"], med["neighbour"], spread["neighbour"], med["call"], spread["call"],
                med["default"], spread["default"]), flush=True)
    return result


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for texture_cost.json (texture_classes_cost.json with --classes)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--classes", default=None,
                    help="comma-separated texture classes, e.g. glcm,glszm,glrlm,gldm,ngtdm: time lm_glrlm_dev and "
                         "lm_neighbour_counts_dev alone and the whole call with these classes instead of the default run")
    args = ap.parse_args()

    import torch
    import bench
    from statistics_cost import gpu_info, lung_mask
    from lungmask_b200 import LMInferer
    from oracle import synth

    info = gpu_info()
    print("gpu: %s" % info)
    sd = bench.get_weights(3, bench.WEIGHT_SEEDS[3])
    fd, wpath = tempfile.mkstemp(suffix=".pth", prefix="texture_cost_")
    os.close(fd)
    try:
        torch.save(sd, wpath)
        inferer = LMInferer(modelname="R231", modelpath=wpath, batch_size=20, tqdm_disable=True, device=0)
    finally:
        os.remove(wpath)
    if args.classes is not None:
        result = classes_cost(inferer, [c.strip() for c in args.classes.split(",") if c.strip()], args.rounds, info)
        if args.out:
            os.makedirs(args.out, exist_ok=True)
            with open(os.path.join(args.out, "texture_classes_cost.json"), "w") as f:
                json.dump(result, f, indent=1)
        return
    rng = np.random.default_rng(100)
    result = {"gpu": info, "workload": "300-slice phantoms seed 100, two-lung ellipsoid mask, GLCM + GLSZM per row",
              "rounds": args.rounds, "unit": "ms", "cases": {}}
    print("\n%-30s %6s %14s %14s %16s %10s" % ("case", "Ng", "device ms", "glcm ms", "numpy-input ms", "host ms"))
    for H in (256, 512):
        base = synth.phantom(SLICES, H, H, seed=100)
        mask = lung_mask(SLICES, H, H)
        for dt in ("int16", "float32"):
            vol = base if dt == "int16" else (base + rng.random(base.shape, dtype=np.float32)).astype(np.float32)
            tv, tm = torch.from_numpy(vol).to("cuda:0"), torch.from_numpy(mask).to("cuda:0")
            for bw in (25, 10):
                name = "%dx%dx%d %s bw %d" % (SLICES, H, H, dt, bw)
                inferer.texture(tv, tm, bin_width=bw)     # warm-up: work buffers, module load
                inferer.texture(vol, mask, bin_width=bw)
                t0 = time.perf_counter()
                want = host_rows(vol, mask, bw)
                host = (time.perf_counter() - t0) * 1e3
                L, ng = want["lung"][2], want["lung"][3]
                tL = torch.from_numpy(L).to("cuda:0")
                dev, glcm, npy = [], [], []
                for _ in range(args.rounds):
                    e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
                    e0.record()
                    r_dev = inferer.texture(tv, tm, bin_width=bw)
                    e1.record()
                    U = inferer.engine.glcm_dev(tL.data_ptr(), L.shape, ng, stream=torch.cuda.current_stream().cuda_stream)
                    e2.record()
                    e2.synchronize()
                    dev.append(e0.elapsed_time(e1))
                    glcm.append(e1.elapsed_time(e2))
                    t0 = time.perf_counter()
                    r_np = inferer.texture(vol, mask, bin_width=bw)
                    npy.append((time.perf_counter() - t0) * 1e3)
                    assert np.array_equal(U, want["lung"][0]), name
                    for row, (Uw, zw, _, _) in want.items():
                        for r in (r_dev, r_np):
                            assert np.array_equal(r[row].glcm_counts, Uw) and np.array_equal(r[row].zones, zw), (name, row)
                med = {k: float(np.median(v)) for k, v in (("device", dev), ("glcm", glcm), ("numpy", npy))}
                spread = {k: float(np.max(v) - np.min(v)) for k, v in (("device", dev), ("glcm", glcm), ("numpy", npy))}
                med["host"] = host
                result["cases"][name] = {"median": med, "spread": spread, "n_levels_lung": ng,
                                         "rounds": {"device": dev, "glcm": glcm, "numpy": npy}}
                print("%-30s %6d %7.2f (%5.2f) %7.2f (%5.2f) %8.1f (%5.1f) %10.0f" % (
                    name, ng, med["device"], spread["device"], med["glcm"], spread["glcm"], med["numpy"], spread["numpy"],
                    host), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "texture_cost.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
