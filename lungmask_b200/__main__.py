"""`lungmask INPUT OUTPUT` command line (flags as lungmask/__main__.py:26-76).

Inputs are read by lungmask_b200/io.py (DICOM series directory, NIfTI, MetaImage, .npy - no SimpleITK needed); the
mask is written with the input's geometry as .nii / .nii.gz / .mha / .npy.  `--probabilities PATH` also writes the
model's per-class probabilities (.npy or 4-D .nii / .nii.gz, LMInferer.apply_with_probabilities), and `--statistics PATH`
the volume and HU statistics of every label and of the whole lung (.json / .csv, LMInferer.statistics: Perc15, LAA-950),
`--clusters PATH` the size distributions of the low-attenuation clusters with their exponent D (.json / .csv,
LMInferer.laa_clusters), and `--regions PATH` the statistics of every label by upper / middle / lower zone and by depth
below the lung surface (.json / .csv, LMInferer.regional_statistics).
"""
import argparse
import os
import sys

from .io import (check_probabilities_path, check_table_path, load_input_image, save_clusters, save_mask, save_probabilities,
                 save_regional_statistics, save_statistics)
from .logger import logger
from .mask import LMInferer

__version__ = "0.1.0+b200"


def _path(string):
    if os.path.exists(string):
        return string
    sys.exit(f"File not found: {string}")


def build_parser():
    p = argparse.ArgumentParser(prog="lungmask")
    p.add_argument("input", metavar="input", type=_path, help="Path to the input image: file, DICOM directory or .npy volume")
    p.add_argument("output", metavar="output", type=str, help="Filepath for output lungmask")
    p.add_argument("--modelname", choices=["R231", "LTRCLobes", "LTRCLobes_R231", "R231CovidWeb"], default="R231")
    p.add_argument("--modelpath", type=str, default=None, help="spcifies the path to the trained model")
    p.add_argument("--cpu", action="store_true", help="not supported by the H100 engine (kept for flag compatibility)")
    p.add_argument("--nopostprocess", action="store_true", help="Deactivates postprocessing")
    p.add_argument("--noHU", action="store_true", help=argparse.SUPPRESS)
    p.add_argument("--batchsize", type=int, default=20, help="Number of slices processed simultaneously")
    p.add_argument("--noprogress", action="store_true", help="If set, no tqdm progress bar will be shown")
    p.add_argument("--version", action="version", version=__version__)
    p.add_argument("--removemetadata", action="store_true", help="Do not keep study/patient metadata of the input")
    p.add_argument("--probabilities", metavar="PATH", type=str, default=None,
                   help="Also write the model's per-class probabilities (before post-processing) with the mask's geometry: "
                        ".npy, or a 4-D .nii / .nii.gz with the classes as 4th dimension. Not for LTRCLobes_R231")
    p.add_argument("--statistics", metavar="PATH", type=str, default=None,
                   help="Also write per-label volume (mL) and HU statistics of the input under the mask - mean, std, min, "
                        "max, Perc15 and LAA-950 - for every label and the whole lung: .json or .csv")
    p.add_argument("--clusters", metavar="PATH", type=str, default=None,
                   help="Also write the size distributions of the connected clusters of low-attenuation voxels (below "
                        "--clusters-threshold HU) for every label and the whole lung, with the power-law exponent D: "
                        ".json (with the (size, count) pairs) or .csv (the summary)")
    p.add_argument("--clusters-threshold", metavar="HU", type=int, default=-950,
                   help="Low-attenuation threshold of --clusters, an integer HU in [-1024, 3072] (default -950)")
    p.add_argument("--clusters-connectivity", type=int, choices=[4, 6, 26], default=6,
                   help="Cluster connectivity of --clusters: 6 faces (default), 26 full, 4 faces within a slice")
    p.add_argument("--regions", metavar="PATH", type=str, default=None,
                   help="Also write the statistics of --statistics for every label and the whole lung by craniocaudal "
                        "zone (upper / middle / lower thirds of each row's volume) and by depth below the lung surface "
                        "(rind < 10 mm, core): .json (with the per-plane volume profile) or .csv")
    return p


def main(argv=None):
    args = build_parser().parse_args(argv)
    if args.probabilities is not None:
        if args.modelname == "LTRCLobes_R231":
            sys.exit("--probabilities: the LTRCLobes_R231 fusion has no class probabilities; use LTRCLobes or R231")
        check_probabilities_path(args.probabilities)
    if args.statistics is not None:
        check_table_path(args.statistics, "statistics")
    if args.clusters is not None:
        check_table_path(args.clusters, "clusters")
        from .clusters import check_arguments
        try:
            check_arguments(args.clusters_threshold, args.clusters_connectivity, 1)
        except ValueError as ex:
            sys.exit("--clusters-threshold: %s" % ex)
    if args.regions is not None:
        check_table_path(args.regions, "regions")
    batchsize = 1 if args.cpu else args.batchsize  # __main__.py:81-83
    logger.info("Load model")
    image = load_input_image(args.input, disable_tqdm=args.noprogress, read_metadata=not args.removemetadata)
    if args.modelname == "LTRCLobes_R231":  # __main__.py:95-107
        assert args.modelpath is None, "Modelpath can not be specified for LTRCLobes_R231 fusion"
        inferer = LMInferer(modelname="LTRCLobes", force_cpu=args.cpu, fillmodel="R231", batch_size=batchsize,
                            volume_postprocessing=not args.nopostprocess, tqdm_disable=args.noprogress)
    else:
        inferer = LMInferer(modelname=args.modelname, modelpath=args.modelpath, force_cpu=args.cpu, batch_size=batchsize,
                            volume_postprocessing=not args.nopostprocess, tqdm_disable=args.noprogress)
    probs = None
    if args.probabilities is None:
        result = inferer.apply(image)  # a Volume: orientation handled as for a SimpleITK image (mask.py:157-164, 189-197)
    else:
        result, probs = inferer.apply_with_probabilities(image)
    logger.info(f"Save result to: {args.output}")
    if not args.removemetadata and image.meta.get("SeriesInstanceUID"):
        logger.info("DICOM tags are never copied into the output by this build (as with --removemetadata)")
    save_mask(args.output, result, image)
    if probs is not None:
        logger.info(f"Save probabilities to: {args.probabilities}")
        save_probabilities(args.probabilities, probs, image)
    if args.statistics is not None:
        logger.info(f"Save statistics to: {args.statistics}")
        save_statistics(args.statistics, inferer.statistics(image, result))
    if args.clusters is not None:
        logger.info(f"Save clusters to: {args.clusters}")
        save_clusters(args.clusters, inferer.laa_clusters(image, result, threshold=args.clusters_threshold,
                                                          connectivity=args.clusters_connectivity))
    if args.regions is not None:
        logger.info(f"Save regional statistics to: {args.regions}")
        save_regional_statistics(args.regions, inferer.regional_statistics(image, result))


if __name__ == "__main__":
    main()
