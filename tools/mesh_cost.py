#!/usr/bin/env python
"""What the surface meshes cost: lm_mesh_counts_dev and lm_mesh_emit_dev per row, LMInferer.mesh on CUDA tensors and on
numpy arrays, and the numpy statement mesh.mesh_host.

    python tools/mesh_cost.py [--out DIR] [--rounds 5]

Builds the engine as bench.py does (R231, the seeded weights of bench.get_weights) and runs, at 300 slices of 256x256 and
512x512, on the two-lung mask of tools/statistics_cost.py (rows 1, 2 and "lung") and on its five-lobe split of
tools/shape_cost.py (rows 1..5 and "lung"), spacing (0.703125, 0.703125, 1.25) mm.  Per case:
  * "counts"  lm_mesh_counts_dev (count pass and offset scan) for every row, CUDA events around each call: the sum over
              the rows and the slowest row
  * "emit"    lm_mesh_emit_dev for every row (it recounts, then writes), the same
  * "device"  LMInferer.mesh on a CUDA tensor, CUDA events on the current stream around the whole call (it synchronises)
  * "numpy"   LMInferer.mesh on the numpy mask, wall time (upload and download of the meshes included)
  * "host"    mesh.mesh_host for every row, one round, wall time
  * V / T     the vertices and triangles of the "lung" row
Median over the rounds and the spread (max - min).  The device meshes are checked bit for bit against mesh_host.  The
card name and power limit come from a read-only nvidia-smi query.  Writes DIR/mesh_cost.json when --out is given.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for mesh_cost.json")
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()

    import torch
    import bench
    from shape_cost import lobes_of
    from statistics_cost import gpu_info, lung_mask
    from lungmask_b200 import LMInferer, mesh as me

    info = gpu_info()
    print("gpu: %s" % info)
    sd = bench.get_weights(3, bench.WEIGHT_SEEDS[3])
    fd, wpath = tempfile.mkstemp(suffix=".pth", prefix="mesh_cost_")
    os.close(fd)
    try:
        torch.save(sd, wpath)
        inferer = LMInferer(modelname="R231", modelpath=wpath, batch_size=20, tqdm_disable=True, device=0)
    finally:
        os.remove(wpath)
    result = {"gpu": info, "workload": "300-slice two-lung ellipsoid mask and its five-lobe split, spacing %s" % (SPACING,),
              "rounds": args.rounds, "unit": "ms", "cases": {}}
    geo = me.geometry_vector(*me.geometry(SPACING))
    off, codes = me.TABLE_OFFSETS, me.TABLE_CODES
    print("\n%-20s %5s %16s %16s %14s %16s %9s  %s" % ("case", "rows", "counts ms (max)", "emit ms (max)", "device ms",
                                                     "numpy-input ms", "host ms", "lung V / T"))
    for H in (256, 512):
        two = lung_mask(SLICES, H, H)
        for which, mask in (("lungs", two), ("lobes", lobes_of(two))):
            name = "%dx%dx%d %s" % (SLICES, H, H, which)
            rows = [int(x) for x in np.unique(mask) if x] + [256]
            tm = torch.from_numpy(mask).to("cuda:0")
            stream = torch.cuda.current_stream().cuda_stream
            inferer.mesh(tm, spacing=SPACING)      # warm-up: work buffers, module load
            inferer.mesh(mask, spacing=SPACING)
            t0 = time.perf_counter()
            want = {r: me.mesh_host(mask, r, SPACING) for r in rows}
            host = (time.perf_counter() - t0) * 1e3
            outs = {r: tuple(torch.empty((n, 3), dtype=dt, device="cuda:0") for n, dt in (
                (want[r].n_vertices, torch.int32), (want[r].n_vertices, torch.float64), (want[r].n_triangles, torch.int32)))
                for r in rows}
            cnt, cnt_max, emit, emit_max, dev, npy = [], [], [], [], [], []
            for _ in range(args.rounds):
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(2 * len(rows) + 2)]
                ev[0].record()
                for k, r in enumerate(rows):
                    nv, nt = inferer.engine.mesh_counts_dev(tm.data_ptr(), mask.shape, r, off, codes, stream=stream)
                    assert (nv, nt) == (want[r].n_vertices, want[r].n_triangles), (name, r)
                    ev[1 + k].record()
                for k, r in enumerate(rows):
                    i2, v, t = outs[r]
                    inferer.engine.mesh_emit_dev(tm.data_ptr(), mask.shape, r, off, codes, geo, want[r].n_vertices,
                                                 want[r].n_triangles, i2.data_ptr(), v.data_ptr(), t.data_ptr(), stream=stream)
                    ev[1 + len(rows) + k].record()
                res = inferer.mesh(tm, spacing=SPACING)
                ev[-1].record()
                ev[-1].synchronize()
                per_c = [ev[k].elapsed_time(ev[k + 1]) for k in range(len(rows))]
                per_e = [ev[len(rows) + k].elapsed_time(ev[len(rows) + k + 1]) for k in range(len(rows))]
                cnt.append(sum(per_c))
                cnt_max.append(max(per_c))
                emit.append(sum(per_e))
                emit_max.append(max(per_e))
                dev.append(ev[-2].elapsed_time(ev[-1]))
                t0 = time.perf_counter()
                res_np = inferer.mesh(mask, spacing=SPACING)
                npy.append((time.perf_counter() - t0) * 1e3)
                for r in rows:
                    label = "lung" if r == 256 else r
                    i2, v, t = outs[r]
                    for got in (res[label].numpy(), res_np[label], me.Mesh(label, "", v.cpu().numpy(), i2.cpu().numpy(),
                                                                           t.cpu().numpy())):
                        assert np.array_equal(got.index2, want[r].index2), (name, r)
                        assert np.array_equal(got.triangles, want[r].triangles), (name, r)
                        assert np.array_equal(got.vertices.view(np.uint64), want[r].vertices.view(np.uint64)), (name, r)
            series = (("counts", cnt), ("counts_max_row", cnt_max), ("emit", emit), ("emit_max_row", emit_max),
                      ("device", dev), ("numpy", npy))
            med = {k: float(np.median(v)) for k, v in series}
            spread = {k: float(np.max(v) - np.min(v)) for k, v in series}
            med["host"] = host
            lung = [want[256].n_vertices, want[256].n_triangles]
            result["cases"][name] = {"median": med, "spread": spread, "rows": rows, "lung_vertices_triangles": lung,
                                     "rounds": {k: v for k, v in series}}
            print("%-20s %5d %7.3f (%6.3f) %7.3f (%6.3f) %7.2f (%4.2f) %8.1f (%5.1f) %9.0f  %d / %d" % (
                name, len(rows), med["counts"], med["counts_max_row"], med["emit"], med["emit_max_row"], med["device"],
                spread["device"], med["numpy"], spread["numpy"], host, *lung), flush=True)
            print("%-20s spread: counts %.3f emit %.3f" % ("", spread["counts"], spread["emit"]), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "mesh_cost.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
