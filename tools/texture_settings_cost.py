#!/usr/bin/env python
"""What PyRadiomics' distances / force2D / weightingNorm settings cost (DESIGN §4.18).

    python tools/texture_settings_cost.py [--out DIR] [--rounds 3] [--sizes 256,512]

Builds the engine as bench.py does (R231, the seeded weights of bench.get_weights) and runs, on the 300-slice int16
phantoms (seed 100) at 256x256 and 512x512 with the two-lung mask of tools/statistics_cost.py, at bin widths 25 and 10,
on the "lung" row's level map:
  * lm_glcm_offsets_dev and lm_neighbour_offsets_dev alone at distances {1} (the 13 offsets of the default path, next
    to lm_glcm_dev and lm_neighbour_counts_dev, alternated within each round), {1,2,3} (171 offsets) and in-plane {1}
    (force2D on axis 0, 4 offsets);
  * lm_zone_sizes_plane_dev (axis 0) next to lm_zone_sizes_dev;
  * the whole LMInferer.texture call with all five classes at {1,2,3}, at force2D axis 0 and at the default settings,
    alternated within each round;
  * the host feature code of GLCM (texture.glcm_features) at 13 and 171 offsets, wall time.
CUDA events around each device call; median over the rounds and the spread (max - min).  Every device matrix is
checked against the numpy references of tests/_texture_settings_ref.py in the same run.  The card name and power
limit come from a read-only nvidia-smi query.  Writes DIR/texture_settings_cost.json when --out is given.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))   # _texture_settings_ref: the numpy references

SLICES = 300


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for texture_settings_cost.json")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sizes", default="256,512", help="in-plane sizes of the phantoms")
    args = ap.parse_args()

    import torch
    import bench
    from statistics_cost import gpu_info, lung_mask
    from _texture_settings_ref import glcm_offsets_ref, neighbour_offsets_ref, plane_structure, zones_ref
    from lungmask_b200 import LMInferer
    from lungmask_b200 import texture as tx
    from oracle import synth

    info = gpu_info()
    print("gpu: %s" % info)
    sd = bench.get_weights(3, bench.WEIGHT_SEEDS[3])
    fd, wpath = tempfile.mkstemp(suffix=".pth", prefix="texture_settings_cost_")
    os.close(fd)
    try:
        torch.save(sd, wpath)
        inferer = LMInferer(modelname="R231", modelpath=wpath, batch_size=20, tqdm_disable=True, device=0)
    finally:
        os.remove(wpath)
    eng = inferer.engine
    sets = {"{1}": tx.offsets((1,)), "{1,2,3}": tx.offsets((1, 2, 3)), "2d {1}": tx.offsets((1,), 0)}
    calls = {"default": {}, "{1,2,3}": dict(distances=(1, 2, 3)), "2d": dict(force2d=True, force2d_dimension=0)}
    result = {"gpu": info, "workload": "300-slice int16 phantoms seed 100, two-lung ellipsoid mask, \"lung\" row",
              "rounds": args.rounds, "unit": "ms", "cases": {}}
    for H in (int(h) for h in args.sizes.split(",")):
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
            tL = torch.from_numpy(L).to("cuda:0")
            p, st = tL.data_ptr(), torch.cuda.current_stream().cuda_stream
            t0 = time.perf_counter()
            want_u = {k: glcm_offsets_ref(L, ng, o) for k, o in sets.items()}
            want_n = {k: neighbour_offsets_ref(L, ng, 0, o) for k, o in sets.items()}
            want_z = zones_ref(L, plane_structure(0))
            ref_s = time.perf_counter() - t0
            jobs = {"glcm_dev": lambda: eng.glcm_dev(p, L.shape, ng, stream=st),
                    "neighbour_counts_dev": lambda: eng.neighbour_counts_dev(p, L.shape, ng, 0, stream=st),
                    "zone_sizes_dev": lambda: eng.zone_sizes_dev(p, L.shape, stream=st),
                    "zone_sizes_plane_dev": lambda: eng.zone_sizes_plane_dev(p, L.shape, 0, stream=st)}
            for k, o in sets.items():
                jobs["glcm_offsets %s" % k] = (lambda o=o: eng.glcm_offsets_dev(p, L.shape, ng, o, stream=st))
                jobs["neighbour_offsets %s" % k] = (lambda o=o: eng.neighbour_offsets_dev(p, L.shape, ng, o, 0, stream=st))
            for k, kw in calls.items():
                jobs["texture %s" % k] = (lambda kw=kw: inferer.texture(tv, tm, bin_width=bw, classes=tx.CLASSES, **kw))
            for job in jobs.values():   # warm-up: work buffers, module load
                job()
            times = {k: [] for k in jobs}
            out = {}
            for _ in range(args.rounds):
                for k, job in jobs.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    out[k] = job()
                    e1.record()
                    e1.synchronize()
                    times[k].append(e0.elapsed_time(e1))
                for k in sets:
                    assert np.array_equal(out["glcm_offsets %s" % k], want_u[k]), (name, k)
                    assert all(np.array_equal(a, b) for a, b in zip(out["neighbour_offsets %s" % k], want_n[k])), (name, k)
                assert np.array_equal(out["glcm_dev"], want_u["{1}"]), name
                assert all(np.array_equal(a, b) for a, b in zip(out["neighbour_counts_dev"], want_n["{1}"])), name
                assert np.array_equal(tx.zones_from_native(out["zone_sizes_plane_dev"]), want_z), name
                r = out["texture {1,2,3}"]["lung"]
                assert np.array_equal(r.glcm_counts, want_u["{1,2,3}"]) and np.array_equal(r.gldm_counts, want_n["{1,2,3}"][0])
                r = out["texture 2d"]["lung"]
                assert np.array_equal(r.glcm_counts, want_u["2d {1}"]) and np.array_equal(r.zones, want_z)
            host = {}
            for k in ("{1}", "{1,2,3}"):
                t0 = time.perf_counter()
                tx.glcm_features(want_u[k], ng)
                host["glcm_features %s" % k] = (time.perf_counter() - t0) * 1e3
            med = {k: float(np.median(v)) for k, v in times.items()}
            spread = {k: float(np.max(v) - np.min(v)) for k, v in times.items()}
            result["cases"][name] = {"n_levels": ng, "median": med, "spread": spread, "rounds": times,
                                     "host_ms": host, "reference_s": ref_s}
            print("\n%s (Ng %d; references %.0f s)" % (name, ng, ref_s))
            for k in jobs:
                print("  %-30s %9.2f ms (spread %.2f)" % (k, med[k], spread[k]))
            for k, v in host.items():
                print("  %-30s %9.2f ms host" % (k, v), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "texture_settings_cost.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
