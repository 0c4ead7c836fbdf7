"""`lungmask INPUT OUTPUT` command line (flags as lungmask/__main__.py:26-76).

Inputs are read by lungmask_b200/io.py (DICOM series directory, NIfTI, MetaImage, .npy - no SimpleITK needed); the
mask is written with the input's geometry as .nii / .nii.gz / .mha / .npy.
"""
import argparse
import os
import sys

from .io import load_input_image, save_mask
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
    return p


def main(argv=None):
    args = build_parser().parse_args(argv)
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
    result = inferer.apply(image)      # a Volume: orientation handled as for a SimpleITK image (mask.py:157-164, 189-197)
    logger.info(f"Save result to: {args.output}")
    if not args.removemetadata and image.meta.get("SeriesInstanceUID"):
        logger.info("DICOM tags are never copied into the output by this build (as with --removemetadata)")
    save_mask(args.output, result, image)


if __name__ == "__main__":
    main()
