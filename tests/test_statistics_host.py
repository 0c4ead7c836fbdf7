"""Host side of the per-label statistics: label names, argument checks, the JSON / CSV writer and the CLI flag."""
import csv
import json
import math

import numpy as np
import pytest


def _stats():
    from lungmask_b200 import statistics as st
    res = {"voxels": np.zeros(257, np.int64), "nan_voxels": np.zeros(257, np.int64), "moments": np.full((257, 4), np.nan),
           "percentile": np.full((257, 2), np.nan), "below_count": np.zeros((257, 1), np.int64)}
    res["voxels"][[1, 256]] = (10, 10)
    res["nan_voxels"][[1, 256]] = (2, 2)
    res["moments"][[1, 256]] = (-850.25, 12.5, -900.0, -700.0)
    res["percentile"][[1, 256]] = (-870.5, -700.0)
    res["below_count"][[1, 256]] = 3
    return st.from_native(res, {1, 2}, "R231", (0.5, 0.5, 2.0), (15.0, 100.0), (-950,))


def test_label_names():
    from lungmask_b200.statistics import label_name
    assert [label_name("R231", l) for l in (1, 2)] == ["right lung", "left lung"]
    assert label_name("R231CovidWeb", 2) == "left lung"
    assert [label_name("LTRCLobes", l) for l in range(1, 6)] == ["left upper lobe", "left lower lobe", "right upper lobe",
                                                                 "right middle lobe", "right lower lobe"]
    assert label_name("LTRCLobes_R231", 4) == "right middle lobe"
    assert label_name("R231", 3) == "label 3" and label_name("w3.pth", 1) == "label 1"


def test_rows():
    s = _stats()
    assert [r.label for r in s.rows] == [1, 2, "lung"] and s["lung"].name == "lung" and s[1].name == "right lung"
    assert s[1].volume_ml == 10 * 0.5 * 0.5 * 2.0 / 1000.0
    assert s[1].fraction_below[-950] == 3 / 8 and s[1].percentile_hu[15.0] == -870.5
    assert s[2].voxels == 0 and math.isnan(s[2].mean_hu) and math.isnan(s[2].fraction_below[-950])
    with pytest.raises(KeyError):
        s[7]


def test_check_arguments():
    from lungmask_b200.statistics import check_arguments
    assert check_arguments((15, 50.5), [-950, 0]) == ((15.0, 50.5), (-950, 0))
    assert check_arguments(15.0, -950) == ((15.0,), (-950,))
    assert check_arguments((), ()) == ((), ())
    assert check_arguments((0.0, 100.0), (-1024, 3072.0)) == ((0.0, 100.0), (-1024, 3072))
    for q in ((-0.1,), (100.5,), (float("nan"),)):
        with pytest.raises(ValueError):
            check_arguments(q, ())
    for t in ((-1025,), (3073,)):
        with pytest.raises(ValueError):
            check_arguments((), t)
    with pytest.raises(TypeError):
        check_arguments((), (-950.5,))
    with pytest.raises(ValueError):
        check_arguments(tuple(range(65)), ())


def test_save_json_and_csv(tmp_path):
    from lungmask_b200 import io as lio
    s = _stats()
    pj, pc = str(tmp_path / "s.json"), str(tmp_path / "s.csv")
    lio.save_statistics(pj, s)
    d = json.load(open(pj))
    assert d["spacing"] == [0.5, 0.5, 2.0] and d["percentiles"] == [15.0, 100.0] and d["thresholds"] == [-950]
    assert [r["label"] for r in d["rows"]] == [1, 2, "lung"]
    assert d["rows"][0]["percentile_hu"] == {"15": -870.5, "100": -700.0} and d["rows"][0]["fraction_below"] == {"-950": 0.375}
    assert d["rows"][1]["mean_hu"] is None and d["rows"][1]["percentile_hu"]["15"] is None   # NaN -> null
    lio.save_statistics(pc, s)
    rows = list(csv.DictReader(open(pc)))
    assert list(rows[0].keys()) == ["label", "name", "voxels", "nan_voxels", "volume_ml", "mean_hu", "std_hu", "min_hu", "max_hu",
                                    "percentile_15", "percentile_100", "fraction_below_-950"]
    assert rows[0]["name"] == "right lung" and int(rows[0]["voxels"]) == 10 and float(rows[0]["volume_ml"]) == s[1].volume_ml
    assert rows[1]["mean_hu"] == "nan" and rows[2]["label"] == "lung"
    with pytest.raises(SystemExit):
        lio.save_statistics(str(tmp_path / "s.txt"), s)


def test_csv_without_spacing(tmp_path):
    from lungmask_b200 import io as lio
    from lungmask_b200 import statistics as st
    s = _stats()
    s2 = st.LabelStatistics(None, s.percentiles, s.thresholds, [st.LabelRow(**{**r.__dict__, "volume_ml": None}) for r in s.rows])
    p = str(tmp_path / "n.csv")
    lio.save_statistics(p, s2)
    assert list(csv.DictReader(open(p)))[0]["volume_ml"] == ""
    lio.save_statistics(str(tmp_path / "n.json"), s2)
    assert json.load(open(str(tmp_path / "n.json")))["spacing"] is None


def test_cli_statistics_flag(tmp_path):
    from lungmask_b200.__main__ import build_parser, main
    inp = tmp_path / "v.npy"
    np.save(inp, np.zeros((2, 8, 8), np.int16))
    args = build_parser().parse_args([str(inp), "out.nii", "--statistics", "s.csv"])
    assert args.statistics == "s.csv"
    assert build_parser().parse_args([str(inp), "out.nii"]).statistics is None
    with pytest.raises(SystemExit, match="statistics"):   # refused before any model is loaded
        main([str(inp), str(tmp_path / "out.nii"), "--statistics", str(tmp_path / "s.xlsx")])
