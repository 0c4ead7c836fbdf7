#!/usr/bin/env python
"""Per-layer times of the 21 tensor-core convolutions of one C2 volume (bench.py's flagship workload).

    python tools/conv_layer_times.py --out DIR [--option conv64_cm --values 1,0,1,0] [--volumes 3]

Builds the engine as bench.py does (R231, the seeded weights of bench.get_weights, the 300-slice phantom with seed 100,
waves of 33 slices), profiles whole-volume forwards with torch.profiler (CUDA activities) after a warm-up, and maps each
convolution kernel record, in start-time order, to its LAYERS index (engine.cu: 21 per wave).  Each entry of --values is
one profiled round with the engine option --option set to it; alternating the settings in one process gives a before /
after that shares the GPU's state.  Prints a table per setting and writes DIR/conv_layer_times.json.

Per kernel it also fits  time = a * tiles + c * k-blocks  over that kernel's 3x3 layers, both counts those of the busiest
CTA (the LAYERS shapes, waves of 33 slices over 132 SMs): c is the mainloop's cost per k-block, a the cost per output tile
that does not overlap it (epilogue, pipeline fill).  The fit is printed for the mean and for every round, whose spread
shows how far a and c can be trusted.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (name, level, C0, C1, Cout, taps) in engine.cu LAYERS order
LAYERS = [
    ("down_path.0.block.3", 0, 64, 0, 64, 9),
    ("down_path.1.block.0", 1, 64, 0, 128, 9),
    ("down_path.1.block.3", 1, 128, 0, 128, 9),
    ("down_path.2.block.0", 2, 128, 0, 256, 9),
    ("down_path.2.block.3", 2, 256, 0, 256, 9),
    ("down_path.3.block.0", 3, 256, 0, 512, 9),
    ("down_path.3.block.3", 3, 512, 0, 512, 9),
    ("down_path.4.block.0", 4, 512, 0, 1024, 9),
    ("down_path.4.block.3", 4, 1024, 0, 1024, 9),
    ("up_path.0.up.1", 4, 1024, 0, 512, 1),
    ("up_path.0.conv_block.block.0", 3, 512, 512, 512, 9),
    ("up_path.0.conv_block.block.3", 3, 512, 0, 512, 9),
    ("up_path.1.up.1", 3, 512, 0, 256, 1),
    ("up_path.1.conv_block.block.0", 2, 256, 256, 256, 9),
    ("up_path.1.conv_block.block.3", 2, 256, 0, 256, 9),
    ("up_path.2.up.1", 2, 256, 0, 128, 1),
    ("up_path.2.conv_block.block.0", 1, 128, 128, 128, 9),
    ("up_path.2.conv_block.block.3", 1, 128, 0, 128, 9),
    ("up_path.3.up.1", 1, 128, 0, 64, 1),
    ("up_path.3.conv_block.block.0", 0, 64, 64, 64, 9),
    ("up_path.3.conv_block.block.3+head", 0, 64, 0, 64, 9),
]
FULL_RES_64 = (0, 19, 20)                                         # the 3x3 layers with 64 output channels at 256x256
LEVEL_1_2_3X3 = [i for i, l in enumerate(LAYERS) if l[1] in (1, 2) and l[5] == 9]
CONV_KERNELS = ("conv_tc_kernel", "conv_cm64_kernel")
RES, SLICES, WAVE = 256, 300, 33
WAVES = [min(WAVE, SLICES - s) for s in range(0, SLICES, WAVE)]   # slices per forward batch
SMS = 132


def layer_gflop(i):
    _, level, c0, c1, cout, taps = LAYERS[i]
    hw = (RES >> level) ** 2
    return 2.0 * hw * cout * (c0 + c1) * taps / 1e9


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or r.stderr.strip()
    except Exception as ex:   # the numbers stay valid without it; say why it is missing
        return "nvidia-smi unavailable: %s" % ex


def conv_records(trace_path):
    with open(trace_path) as f:
        ev = json.load(f)["traceEvents"]
    ks = [e for e in ev if e.get("cat") == "kernel" and any(k in e.get("name", "") for k in CONV_KERNELS)]
    ks.sort(key=lambda e: e["ts"])
    return [(e["name"], float(e["dur"]) * 1e-3) for e in ks]   # ms


def profile_round(eng, run_volume, volumes):
    """ms per volume of every LAYERS index, averaged over `volumes` profiled forwards, and the kernel name per layer"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(volumes):
            run_volume()
        torch.cuda.synchronize()
    fd, path = tempfile.mkstemp(suffix=".json", prefix="conv_layer_times_")
    os.close(fd)
    try:
        prof.export_chrome_trace(path)
        recs = conv_records(path)
    finally:
        os.remove(path)
    waves = -(-SLICES // WAVE) * volumes
    if len(recs) != waves * len(LAYERS):
        raise SystemExit("expected %d convolution kernel records (%d waves x %d layers), found %d"
                         % (waves * len(LAYERS), waves, len(LAYERS), len(recs)))
    ms = np.zeros(len(LAYERS))
    names = [None] * len(LAYERS)
    for k, (name, dur) in enumerate(recs):
        i = k % len(LAYERS)
        ms[i] += dur
        m = re.search(r"conv_\w*kernel(<[^>]*>)?", name)
        names[i] = m.group(0) if m else name
    return ms / volumes, names


def table(ms, names):
    rows = []
    for i, (lname, level, c0, c1, cout, taps) in enumerate(LAYERS):
        gf = layer_gflop(i) * SLICES
        rows.append({"layer": i, "name": lname, "shape": "%dx%d %d%s->%d %dx%d" % (RES >> level, RES >> level, c0,
                     "+%d" % c1 if c1 else "", cout, 3 if taps == 9 else 1, 3 if taps == 9 else 1),
                     "gflop_per_slice": layer_gflop(i), "ms_per_volume": float(ms[i]),
                     "tflops": gf / (ms[i] * 1e-3) / 1e3, "kernel": names[i]})
    return rows


def launch_work(i, kernel):
    """(tiles, k-blocks) of the busiest CTA of layer i, summed over one volume's waves: conv_tc_kernel<BN, MC> tiles are
    16x8 pixels x BN channels, conv_cm64_kernel tiles 16x16 pixels x 64 channels; a launch spreads its tiles over SMS CTAs"""
    _, level, c0, c1, cout, taps = LAYERS[i]
    hw = RES >> level
    if "cm64" in kernel:
        tiles_per_image = (hw // 16) ** 2
    else:
        bn = int(re.search(r"<\s*(\d+)", kernel).group(1))
        tiles_per_image = (hw // 16) * (hw // 8) * (cout // bn)
    kb_per_tile = (c0 + c1) // 64 * taps
    tiles = sum(-(-n * tiles_per_image // SMS) for n in WAVES)
    return tiles, tiles * kb_per_tile


def tile_fit(ms, names):
    """per kernel, the least-squares fit  us per volume = a * tiles per CTA + c * k-blocks per CTA  over its 3x3 layers"""
    fits = {}
    for kernel in sorted(set(names)):
        idx = [i for i in range(len(LAYERS)) if names[i] == kernel and LAYERS[i][5] == 9]
        if len(idx) < 2:
            continue
        X = np.array([launch_work(i, kernel) for i in idx], dtype=float)
        y = np.array([ms[i] * 1e3 for i in idx])
        (a, c), *_ = np.linalg.lstsq(X, y, rcond=None)
        fits[kernel] = {"layers": idx, "a_us_per_tile": float(a), "c_us_per_kblock": float(c),
                        "per_tile_share": float(a * X[:, 0].sum() / y.sum())}
    return fits


def print_fit(fits, per_round):
    for kernel, f in fits.items():
        rounds = [r[kernel] for r in per_round if kernel in r]
        print("%-24s a = %6.2f us/tile (rounds %s), c = %6.3f us/k-block (rounds %s); per-tile term %.1f %% of its time"
              % (kernel, f["a_us_per_tile"], ", ".join("%.2f" % r["a_us_per_tile"] for r in rounds), f["c_us_per_kblock"],
                 ", ".join("%.3f" % r["c_us_per_kblock"] for r in rounds), 100 * f["per_tile_share"]))


def summary(rows):
    def tf(idx):
        return sum(rows[i]["gflop_per_slice"] for i in idx) * SLICES / (sum(rows[i]["ms_per_volume"] for i in idx) * 1e-3) / 1e3
    total = sum(r["ms_per_volume"] for r in rows)
    fr = sum(rows[i]["ms_per_volume"] for i in FULL_RES_64)
    return {"conv_ms_per_volume": total, "full_res_64_ms": fr, "full_res_64_share": fr / total,
            "full_res_64_tflops": tf(FULL_RES_64), "level_1_2_3x3_tflops": tf(LEVEL_1_2_3X3)}


def print_table(label, rows, summ):
    print("\n== %s" % label)
    print("%3s %-36s %-22s %7s %9s %8s  %s" % ("idx", "layer", "shape", "GFLOP/s", "ms/vol", "TFLOP/s", "kernel"))
    for r in rows:
        print("%3d %-36s %-22s %7.2f %9.3f %8.1f  %s" % (r["layer"], r["name"], r["shape"], r["gflop_per_slice"],
                                                        r["ms_per_volume"], r["tflops"], r["kernel"]))
    print("convolutions %.3f ms/volume; layers 0, 19, 20: %.3f ms (%.1f %%), %.1f TFLOP/s; 3x3 layers of levels 1-2: %.1f TFLOP/s"
          % (summ["conv_ms_per_volume"], summ["full_res_64_ms"], 100 * summ["full_res_64_share"],
             summ["full_res_64_tflops"], summ["level_1_2_3x3_tflops"]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for conv_layer_times.json")
    ap.add_argument("--option", default="conv64_cm", help="engine option alternated between rounds ('' = defaults only)")
    ap.add_argument("--values", default="1,0,1,0", help="the option's value in each profiled round")
    ap.add_argument("--volumes", type=int, default=3, help="profiled volume forwards per round")
    ap.add_argument("--warmup", type=int, default=2, help="volume forwards before each round")
    args = ap.parse_args()

    import torch
    import bench
    from lungmask_b200 import LMInferer
    from oracle import synth

    info = gpu_info()
    print("gpu: %s" % info)
    sd = bench.get_weights(3, bench.WEIGHT_SEEDS[3])
    fd, wpath = tempfile.mkstemp(suffix=".pth", prefix="conv_layer_times_")
    os.close(fd)
    try:
        torch.save(sd, wpath)
        inferer = LMInferer(modelname="R231", modelpath=wpath, batch_size=20, tqdm_disable=True, device=0)
    finally:
        os.remove(wpath)
    assert inferer.wave_slices == WAVE, inferer.wave_slices
    eng = inferer.engine
    eng.set_option("graphs", 0)   # one launch per kernel: the records map to layers without relying on graph tracing
    vol = synth.phantom(SLICES, seed=100)
    d_vol = torch.from_numpy(vol).cuda()
    d_out = torch.empty(vol.shape, dtype=torch.uint8, device="cuda")

    def run_volume():
        eng.apply_volume_dev(0, d_vol.data_ptr(), vol.shape, d_out.data_ptr())

    values = [int(v) for v in args.values.split(",")] if args.option else [None]
    rounds = []
    for v in values:
        if v is not None:
            eng.set_option(args.option, v)
        for _ in range(args.warmup):
            run_volume()
        torch.cuda.synchronize()
        ms, names = profile_round(eng, run_volume, args.volumes)
        rounds.append({"value": v, "ms": ms, "names": names})

    result = {"gpu": info, "workload": "C2: R231 (3 classes), 300-slice 256x256 phantom seed 100, waves of %d" % WAVE,
              "option": args.option or None, "rounds": [r["value"] for r in rounds], "volumes_per_round": args.volumes,
              "settings": {}}
    for v in sorted({r["value"] for r in rounds}, key=lambda x: (x is None, x)):
        mine = [r for r in rounds if r["value"] == v]
        ms = np.mean([r["ms"] for r in mine], axis=0)
        spread = np.max([r["ms"] for r in mine], axis=0) - np.min([r["ms"] for r in mine], axis=0)
        rows = table(ms, mine[0]["names"])
        for r, s in zip(rows, spread):
            r["ms_spread_between_rounds"] = float(s)
        summ = summary(rows)
        summ["full_res_64_ms_per_round"] = [float(sum(r["ms"][i] for i in FULL_RES_64)) for r in mine]
        label = "defaults" if v is None else "%s = %d" % (args.option, v)
        print_table(label, rows, summ)
        fits = tile_fit(ms, mine[0]["names"])
        per_round = [tile_fit(r["ms"], r["names"]) for r in mine]
        print_fit(fits, per_round)
        result["settings"][label] = {"layers": rows, "summary": summ, "tile_fit": fits, "tile_fit_per_round": per_round}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "conv_layer_times.json"), "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
