"""`lungmask INPUT OUTPUT` command line (flags as lungmask/__main__.py:26-76).

Inputs are read by lungmask_b200/io.py (DICOM series directory, NIfTI, MetaImage, .npy - no SimpleITK needed); the
mask is written with the input's geometry as .nii / .nii.gz / .mha / .npy.  `--probabilities PATH` also writes the
model's per-class probabilities (.npy or 4-D .nii / .nii.gz, LMInferer.apply_with_probabilities), and `--statistics PATH`
the volume and HU statistics of every label and of the whole lung (.json / .csv, LMInferer.statistics: Perc15, LAA-950),
`--clusters PATH` the size distributions of the low-attenuation clusters with their exponent D (.json / .csv,
LMInferer.laa_clusters), `--regions PATH` the statistics of every label by upper / middle / lower zone and by depth
below the lung surface (.json / .csv, LMInferer.regional_statistics), `--texture PATH` the texture features of every
label and the whole lung (GLCM and GLSZM by default, `--texture-classes` adds GLRLM, GLDM and NGTDM; .json / .csv,
LMInferer.texture), `--shape PATH` the mesh shape features
(surface area, mesh volume, sphericity, maximum diameters, principal axes) of every label and the whole lung (.json /
.csv, LMInferer.shape), and `--first-order PATH` PyRadiomics' first-order features (percentiles, moments, mean absolute
deviations, energy, entropy, uniformity) of every label and the whole lung (.json / .csv, LMInferer.first_order), and
`--wavelet PATH` the first-order and texture features of the 8 coif1 (or haar) wavelet decompositions (.json / .csv,
LMInferer.wavelet_features), and `--filtered PATH` those of the Square, SquareRoot, Logarithm, Exponential and Gradient
image types (.json / .csv, LMInferer.filtered_features), and `--log PATH` those of the LoG image type at each sigma of
`--log-sigma` (.json / .csv, LMInferer.log_features), and `--mesh DIR` the marching-cubes surface of every present
label and of the whole lung, one file per row (`--mesh-format` stl, obj or ply, `--mesh-space` lps or ras;
LMInferer.mesh with the input's geometry), and `--first-order-maps DIR` the voxel-based first-order feature maps of one
row, one image per feature with the input's geometry (LMInferer.first_order_maps), and `--glcm-maps DIR` its voxel-based
GLCM feature maps the same way (LMInferer.glcm_maps), and `--texture-maps DIR` its voxel-based GLSZM, GLRLM, GLDM and
NGTDM feature maps (LMInferer.texture_maps).  `--texture-distances`, `--texture-force2d` and `--texture-weighting-norm`
set PyRadiomics' distances, force2D and weightingNorm for the texture matrices of --texture, --wavelet, --filtered and
--log.
`--resample X,Y,Z` resamples the image and the mask once after segmentation to that spacing in mm (PyRadiomics'
resampledPixelSpacing, `--resample-interpolator` bspline or nearest; LMInferer.resample), and --texture, --shape,
--first-order, --wavelet, --filtered and --log then run on the resampled pair; the other analyses stay on the native
grid.
"""
import argparse
import os
import sys

from .io import (check_probabilities_path, check_table_path, load_input_image, save_clusters, save_first_order, save_mask,
                 save_feature_maps, save_mesh, save_probabilities, save_regional_statistics, save_shape, save_statistics, save_texture,
                 save_filtered_features, save_log_features, save_wavelet_features)
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
    p.add_argument("--texture", metavar="PATH", type=str, default=None,
                   help="Also write the texture features (PyRadiomics names) of every label and the whole lung, of the "
                        "classes of --texture-classes: .json (with the exact matrices) or .csv")
    p.add_argument("--texture-bin-width", metavar="BW", type=int, default=25,
                   help="Fixed bin width of --texture in HU, a positive integer (default 25)")
    p.add_argument("--texture-classes", metavar="NAMES", type=str, default="glcm,glszm",
                   help="Comma-separated texture classes of --texture: any of glcm, glszm, glrlm, gldm, ngtdm "
                        "(default glcm,glszm)")
    p.add_argument("--texture-distances", metavar="D", type=str, default=None,
                   help="Comma-separated neighbour distances 1..3 of the GLCM, GLDM and NGTDM of --texture, --wavelet and "
                        "--filtered, such as 1,2,3 (PyRadiomics' distances; default 1)")
    p.add_argument("--texture-force2d", metavar="AXIS", type=int, choices=[0, 1, 2], default=None,
                   help="Texture matrices of --texture, --wavelet and --filtered within the planes normal to array axis "
                        "AXIS (0: axial slices; PyRadiomics' force2D / force2Ddimension; default 3-D)")
    p.add_argument("--texture-weighting-norm", choices=["manhattan", "euclidean", "infinity", "no_weighting"], default=None,
                   help="Merge the GLCM and GLRLM matrices of --texture, --wavelet and --filtered over directions with "
                        "spacing-based weights before computing features (PyRadiomics' weightingNorm; default: features "
                        "averaged over directions)")
    p.add_argument("--shape", metavar="PATH", type=str, default=None,
                   help="Also write the mesh shape features (PyRadiomics names: surface area, mesh volume, sphericity, "
                        "maximum 3-D and 2-D diameters, principal axis lengths) of every label and the whole lung: .json "
                        "(with the exact sums) or .csv")
    p.add_argument("--first-order", metavar="PATH", type=str, default=None,
                   help="Also write the first-order features (PyRadiomics names: percentiles, mean, variance, skewness, "
                        "kurtosis, mean absolute deviations, energy, entropy, uniformity) of every label and the whole "
                        "lung: .json (with the level histograms and the exact sums) or .csv")
    p.add_argument("--first-order-bin-width", metavar="BW", type=int, default=25,
                   help="Fixed bin width of the Entropy and Uniformity of --first-order in HU, a positive integer "
                        "(default 25)")
    p.add_argument("--first-order-shift", metavar="C", type=int, default=0,
                   help="Integer added to every value for Energy, TotalEnergy and RootMeanSquared of --first-order "
                        "(PyRadiomics' voxelArrayShift, default 0)")
    p.add_argument("--wavelet", metavar="PATH", type=str, default=None,
                   help="Also write the first-order and texture features of the 8 wavelet decompositions (PyRadiomics' "
                        "Wavelet image type, keys such as wavelet-LLH_firstorder_Mean) of every label and the whole lung: "
                        ".json (with the exact sums and matrices) or .csv")
    p.add_argument("--wavelet-name", choices=["coif1", "haar"], default="coif1", help="Wavelet of --wavelet (default coif1)")
    p.add_argument("--wavelet-bin-width", metavar="SPEC", type=str, default="25",
                   help="Fixed bin width of --wavelet in HU: one positive integer, or a default followed by "
                        "per-decomposition overrides such as 25,LLL=50 (default 25)")
    p.add_argument("--wavelet-classes", metavar="NAMES", type=str, default="firstorder,glcm,glszm,glrlm,gldm,ngtdm",
                   help="Comma-separated feature classes of --wavelet: any of firstorder, glcm, glszm, glrlm, gldm, ngtdm "
                        "(default all)")
    p.add_argument("--filtered", metavar="PATH", type=str, default=None,
                   help="Also write the first-order and texture features of PyRadiomics' Square, SquareRoot, Logarithm, "
                        "Exponential and Gradient image types (keys such as square_firstorder_Mean) of every label and the "
                        "whole lung: .json (with the exact sums and matrices) or .csv")
    p.add_argument("--filtered-types", metavar="NAMES", type=str,
                   default="square,squareroot,logarithm,exponential,gradient",
                   help="Comma-separated image types of --filtered: any of square, squareroot, logarithm, exponential, "
                        "gradient (default all)")
    p.add_argument("--filtered-bin-width", metavar="SPEC", type=str, default="25",
                   help="Fixed bin width of --filtered: one positive integer, or a default followed by per-type overrides "
                        "such as 25,gradient=10 (default 25)")
    p.add_argument("--filtered-classes", metavar="NAMES", type=str, default="firstorder,glcm,glszm,glrlm,gldm,ngtdm",
                   help="Comma-separated feature classes of --filtered: any of firstorder, glcm, glszm, glrlm, gldm, "
                        "ngtdm (default all)")
    p.add_argument("--log", metavar="PATH", type=str, default=None,
                   help="Also write the first-order and texture features of PyRadiomics' LoG image type at each sigma of "
                        "--log-sigma (keys such as log-sigma-1-0-mm-3D_firstorder_Mean) of every label and the whole "
                        "lung: .json (with the exact sums and matrices) or .csv")
    p.add_argument("--log-sigma", metavar="SIGMAS", type=str, default=None,
                   help="Comma-separated sigmas of --log in mm, such as 1,2,3,4,5 (PyRadiomics' LoG sigma; required with "
                        "--log)")
    p.add_argument("--log-bin-width", metavar="SPEC", type=str, default="25",
                   help="Fixed bin width of --log: one positive integer, or a default followed by per-sigma overrides "
                        "such as 25,3.0=50 (default 25)")
    p.add_argument("--log-classes", metavar="NAMES", type=str, default="firstorder,glcm,glszm,glrlm,gldm,ngtdm",
                   help="Comma-separated feature classes of --log: any of firstorder, glcm, glszm, glrlm, gldm, ngtdm "
                        "(default all)")
    p.add_argument("--mesh", metavar="DIR", type=str, default=None,
                   help="Also write the marching-cubes surface (the mesh of --shape, in patient space) of every present "
                        "label and of the whole lung to DIR, one file per row named after it (right_lung.stl, lung.stl)")
    p.add_argument("--mesh-format", choices=["stl", "obj", "ply"], default="stl",
                   help="File format of --mesh: binary STL (default), ASCII OBJ or binary PLY")
    p.add_argument("--mesh-space", choices=["lps", "ras"], default="lps",
                   help="Frame of the --mesh positions: LPS (DICOM / ITK, default) or RAS (3D Slicer, NIfTI)")
    p.add_argument("--first-order-maps", metavar="DIR", type=str, default=None,
                   help="Also write voxel-based first-order feature maps (PyRadiomics' voxelBased extraction) of one row "
                        "to DIR, one float64 image per feature named <row>_<Feature> (lung_Entropy.nii.gz); uses "
                        "--first-order-bin-width and --first-order-shift")
    p.add_argument("--first-order-maps-radius", type=int, choices=[1, 2, 3], default=1,
                   help="Kernel radius of --first-order-maps: the window is the (2r+1)^3 cube about each voxel (default 1)")
    p.add_argument("--first-order-maps-features", metavar="NAMES", type=str, default=None,
                   help="Comma-separated features of --first-order-maps, PyRadiomics names such as Mean,Entropy "
                        "(default all 18)")
    p.add_argument("--first-order-maps-label", metavar="ROW", type=str, default="lung",
                   help='Row of --first-order-maps: "lung" (every label, default) or one label value 1..255')
    p.add_argument("--first-order-maps-unmasked", action="store_true",
                   help="Windows of --first-order-maps take every non-NaN voxel, not only the row's (PyRadiomics' "
                        "maskedKernel=False)")
    p.add_argument("--first-order-maps-format", choices=["nii.gz", "nii", "mha", "npy"], default="nii.gz",
                   help="File format of --first-order-maps (default nii.gz)")
    p.add_argument("--glcm-maps", metavar="DIR", type=str, default=None,
                   help="Also write voxel-based GLCM feature maps (PyRadiomics' voxelBased extraction) of one row to DIR, "
                        "one float64 image per feature named <row>_glcm_<Feature> (lung_glcm_Contrast.nii.gz); uses "
                        "--texture-bin-width")
    p.add_argument("--glcm-maps-radius", type=int, choices=[1, 2, 3], default=1,
                   help="Kernel radius of --glcm-maps: the window is the (2r+1)^3 cube about each voxel (default 1)")
    p.add_argument("--glcm-maps-features", metavar="NAMES", type=str, default=None,
                   help="Comma-separated features of --glcm-maps, PyRadiomics names such as Contrast,JointEntropy,Idm "
                        "(default all 22)")
    p.add_argument("--glcm-maps-label", metavar="ROW", type=str, default="lung",
                   help='Row of --glcm-maps: "lung" (every label, default) or one label value 1..255')
    p.add_argument("--glcm-maps-unmasked", action="store_true",
                   help="Windows of --glcm-maps take every non-NaN voxel, not only the row's (PyRadiomics' "
                        "maskedKernel=False)")
    p.add_argument("--glcm-maps-format", choices=["nii.gz", "nii", "mha", "npy"], default="nii.gz",
                   help="File format of --glcm-maps (default nii.gz)")
    p.add_argument("--texture-maps", metavar="DIR", type=str, default=None,
                   help="Also write voxel-based GLSZM, GLRLM, GLDM and NGTDM feature maps (PyRadiomics' voxelBased "
                        "extraction) of one row to DIR, one float64 image per feature named <row>_<class>_<Feature> "
                        "(lung_glszm_ZoneEntropy.nii.gz); uses --texture-bin-width")
    p.add_argument("--texture-maps-classes", metavar="NAMES", type=str, default="glszm,glrlm,gldm,ngtdm",
                   help="Comma-separated classes of --texture-maps: any of glszm, glrlm, gldm, ngtdm (default all; GLCM "
                        "maps come from --glcm-maps)")
    p.add_argument("--texture-maps-radius", type=int, choices=[1, 2, 3], default=1,
                   help="Kernel radius of --texture-maps: the window is the (2r+1)^3 cube about each voxel (default 1)")
    p.add_argument("--texture-maps-features", metavar="NAMES", type=str, default=None,
                   help="Comma-separated features of --texture-maps, class-qualified PyRadiomics names such as "
                        "glszm_ZoneEntropy,ngtdm_Contrast (default every feature of --texture-maps-classes)")
    p.add_argument("--texture-maps-label", metavar="ROW", type=str, default="lung",
                   help='Row of --texture-maps: "lung" (every label, default) or one label value 1..255')
    p.add_argument("--texture-maps-unmasked", action="store_true",
                   help="Windows of --texture-maps take every non-NaN voxel, not only the row's (PyRadiomics' "
                        "maskedKernel=False)")
    p.add_argument("--texture-maps-format", choices=["nii.gz", "nii", "mha", "npy"], default="nii.gz",
                   help="File format of --texture-maps (default nii.gz)")
    p.add_argument("--resample", metavar="X,Y,Z", type=str, default=None,
                   help="Resample the image and the mask to this spacing in mm (0 keeps an axis; PyRadiomics' "
                        "resampledPixelSpacing) before --texture, --shape, --first-order, --wavelet, --filtered and --log. "
                        "--statistics, --clusters, --regions, --mesh and the feature maps stay on the native grid")
    p.add_argument("--resample-interpolator", choices=["bspline", "nearest"], default=None,
                   help="Image interpolator of --resample: cubic B-spline (sitkBSpline, default) or nearest neighbour; "
                        "the mask is always resampled by nearest neighbour")
    return p


RESAMPLED_ANALYSES = ("texture", "shape", "first_order", "wavelet", "filtered", "log")   # the flags --resample applies to


def resample_arguments(args):
    """-> (resampled spacing (x, y, z), interpolator) of --resample, or None without it; exits with a message naming the
    flag for a bad value."""
    from .resample import parse_spacing
    if args.resample is None:
        if args.resample_interpolator is not None:
            sys.exit("--resample-interpolator: needs --resample")
        return None
    try:
        spacing = parse_spacing(args.resample)
    except ValueError as ex:
        sys.exit("--resample: %s" % ex)
    if all(getattr(args, a) is None for a in RESAMPLED_ANALYSES):
        sys.exit("--resample: applies to --texture, --shape, --first-order, --wavelet, --filtered and --log, and none "
                 "is given")
    return spacing, args.resample_interpolator or "bspline"


def log_arguments(args):
    """-> (sigmas, bin widths, classes) of --log, or None without it; exits with a message naming the flag for a bad
    value."""
    from . import laplacian
    if args.log is None:
        if args.log_sigma is not None:
            sys.exit("--log-sigma: needs --log")
        return None
    check_table_path(args.log, "log")
    if args.log_sigma is None:
        sys.exit("--log: needs --log-sigma, such as --log-sigma 1,2,3,4,5 (PyRadiomics has no default sigma)")
    try:
        sigmas = laplacian.parse_sigmas(args.log_sigma)
    except (TypeError, ValueError) as ex:
        sys.exit("--log-sigma: %s" % ex)
    try:
        widths = laplacian.parse_bin_widths(args.log_bin_width, sigmas)
    except (TypeError, ValueError) as ex:
        sys.exit("--log-bin-width: %s" % ex)
    classes = [c.strip() for c in args.log_classes.split(",") if c.strip()]
    try:
        laplacian.check_classes(classes)
    except (TypeError, ValueError) as ex:
        sys.exit("--log-classes: %s" % ex)
    return sigmas, widths, classes


def texture_settings_arguments(args):
    """-> the keyword arguments distances, force2d, force2d_dimension, weighting_norm of the --texture-* settings;
    exits with a message naming the flag for a bad value."""
    from .texture import check_settings
    distances = (1,)
    if args.texture_distances is not None:
        try:
            distances = [int(c.strip()) for c in args.texture_distances.split(",") if c.strip()]
            check_settings(distances)
        except (TypeError, ValueError) as ex:
            sys.exit("--texture-distances: %s" % ex)
    return {"distances": tuple(distances), "force2d": args.texture_force2d is not None,
            "force2d_dimension": args.texture_force2d or 0, "weighting_norm": args.texture_weighting_norm}


def first_order_maps_arguments(args):
    """-> (label, features) of --first-order-maps; exits with a message naming the flag for a bad value."""
    from . import first_order_maps as fm
    from .texture import check_arguments as check_bin_width
    if os.path.exists(args.first_order_maps) and not os.path.isdir(args.first_order_maps):
        sys.exit("--first-order-maps: %s exists and is not a directory" % args.first_order_maps)
    if not os.path.isdir(os.path.dirname(os.path.abspath(args.first_order_maps))):
        sys.exit("--first-order-maps: the parent directory of %s does not exist" % args.first_order_maps)
    try:
        check_bin_width(args.first_order_bin_width)
    except ValueError as ex:
        sys.exit("--first-order-bin-width: %s" % ex)
    label = args.first_order_maps_label.strip()
    try:
        label = fm.check_label(label if label == "lung" else int(label))
    except ValueError as ex:
        sys.exit("--first-order-maps-label: %s" % ex)
    features = None
    if args.first_order_maps_features is not None:
        try:
            features = fm.check_features([c.strip() for c in args.first_order_maps_features.split(",") if c.strip()])
        except ValueError as ex:
            sys.exit("--first-order-maps-features: %s" % ex)
    return label, features


def glcm_maps_arguments(args):
    """-> (label, features) of --glcm-maps; exits with a message naming the flag for a bad value."""
    from . import first_order_maps as fm
    from . import glcm_maps as gm
    from .texture import check_arguments as check_bin_width
    if os.path.exists(args.glcm_maps) and not os.path.isdir(args.glcm_maps):
        sys.exit("--glcm-maps: %s exists and is not a directory" % args.glcm_maps)
    if not os.path.isdir(os.path.dirname(os.path.abspath(args.glcm_maps))):
        sys.exit("--glcm-maps: the parent directory of %s does not exist" % args.glcm_maps)
    try:
        check_bin_width(args.texture_bin_width)
    except (TypeError, ValueError) as ex:
        sys.exit("--texture-bin-width: %s" % ex)
    label = args.glcm_maps_label.strip()
    try:
        label = fm.check_label(label if label == "lung" else int(label))
    except ValueError as ex:
        sys.exit("--glcm-maps-label: %s" % ex)
    features = None
    if args.glcm_maps_features is not None:
        try:
            features = gm.check_features([c.strip() for c in args.glcm_maps_features.split(",") if c.strip()])
        except ValueError as ex:
            sys.exit("--glcm-maps-features: %s" % ex)
    return label, features


def texture_maps_arguments(args):
    """-> (label, classes, features) of --texture-maps; exits with a message naming the flag for a bad value."""
    from . import first_order_maps as fm
    from . import texture_maps as tm
    from .texture import check_arguments as check_bin_width
    if os.path.exists(args.texture_maps) and not os.path.isdir(args.texture_maps):
        sys.exit("--texture-maps: %s exists and is not a directory" % args.texture_maps)
    if not os.path.isdir(os.path.dirname(os.path.abspath(args.texture_maps))):
        sys.exit("--texture-maps: the parent directory of %s does not exist" % args.texture_maps)
    try:
        check_bin_width(args.texture_bin_width)
    except (TypeError, ValueError) as ex:
        sys.exit("--texture-bin-width: %s" % ex)
    label = args.texture_maps_label.strip()
    try:
        label = fm.check_label(label if label == "lung" else int(label))
    except ValueError as ex:
        sys.exit("--texture-maps-label: %s" % ex)
    try:
        classes = tm.check_classes([c.strip() for c in args.texture_maps_classes.split(",") if c.strip()])
    except ValueError as ex:
        sys.exit("--texture-maps-classes: %s" % ex)
    features = None
    if args.texture_maps_features is not None:
        try:
            features = tm.check_features([c.strip() for c in args.texture_maps_features.split(",") if c.strip()], classes)
        except ValueError as ex:
            sys.exit("--texture-maps-features: %s" % ex)
    return label, classes, features


def mesh_file_name(mesh, fmt):
    """The file --mesh writes a row's mesh to: its name with spaces as underscores."""
    return "%s.%s" % (str(mesh.name).replace(" ", "_"), fmt)


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
    if args.texture is not None:
        check_table_path(args.texture, "texture")
        from .texture import check_arguments as check_texture_arguments, check_classes
        try:
            check_texture_arguments(args.texture_bin_width)
        except ValueError as ex:
            sys.exit("--texture-bin-width: %s" % ex)
        try:
            texture_classes = check_classes([c.strip() for c in args.texture_classes.split(",") if c.strip()])
        except ValueError as ex:
            sys.exit("--texture-classes: %s" % ex)
    settings = texture_settings_arguments(args)
    if args.shape is not None:
        check_table_path(args.shape, "shape")
    if args.first_order is not None:
        check_table_path(args.first_order, "first_order")
        from .texture import check_arguments as check_bin_width
        try:
            check_bin_width(args.first_order_bin_width)
        except ValueError as ex:
            sys.exit("--first-order-bin-width: %s" % ex)
    if args.wavelet is not None:
        check_table_path(args.wavelet, "wavelet")
        from .wavelet import check_classes as check_wavelet_classes, parse_bin_widths
        try:
            wavelet_bin_width = parse_bin_widths(args.wavelet_bin_width)
        except (TypeError, ValueError) as ex:
            sys.exit("--wavelet-bin-width: %s" % ex)
        wavelet_classes = [c.strip() for c in args.wavelet_classes.split(",") if c.strip()]
        try:
            check_wavelet_classes(wavelet_classes)
        except ValueError as ex:
            sys.exit("--wavelet-classes: %s" % ex)
    if args.filtered is not None:
        check_table_path(args.filtered, "filtered")
        from . import filters
        filtered_types = [c.strip() for c in args.filtered_types.split(",") if c.strip()]
        try:
            filtered_types = filters.check_image_types(filtered_types)
        except ValueError as ex:
            sys.exit("--filtered-types: %s" % ex)
        try:
            filtered_bin_width = filters.check_bin_widths(filters.parse_bin_widths(args.filtered_bin_width), filtered_types)
        except (TypeError, ValueError) as ex:
            sys.exit("--filtered-bin-width: %s" % ex)
        filtered_classes = [c.strip() for c in args.filtered_classes.split(",") if c.strip()]
        try:
            filters.check_classes(filtered_classes)
        except ValueError as ex:
            sys.exit("--filtered-classes: %s" % ex)
    if args.mesh is not None:
        if os.path.exists(args.mesh) and not os.path.isdir(args.mesh):
            sys.exit("--mesh: %s exists and is not a directory" % args.mesh)
        parent = os.path.dirname(os.path.abspath(args.mesh))
        if not os.path.isdir(parent):
            sys.exit("--mesh: the parent directory of %s does not exist" % args.mesh)
    if args.first_order_maps is not None:
        maps_label, maps_features = first_order_maps_arguments(args)
    if args.glcm_maps is not None:
        glcm_label, glcm_features = glcm_maps_arguments(args)
    if args.texture_maps is not None:
        tmaps_label, tmaps_classes, tmaps_features = texture_maps_arguments(args)
    log = log_arguments(args)
    resampling = resample_arguments(args)
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
    feature_image, feature_mask = image, result   # the pair of --texture, --shape, --first-order, --wavelet, --filtered, --log
    if resampling is not None:
        logger.info("Resample to %s mm (%s)" % (",".join("%g" % v for v in resampling[0]), resampling[1]))
        r = inferer.resample(image, result, resampled_spacing=resampling[0], interpolator=resampling[1])
        feature_image, feature_mask = r.volume(), r.mask
    if args.texture is not None:
        logger.info(f"Save texture features to: {args.texture}")
        save_texture(args.texture, inferer.texture(feature_image, feature_mask, bin_width=args.texture_bin_width, classes=texture_classes,
                                                           **settings))
    if args.shape is not None:
        logger.info(f"Save shape features to: {args.shape}")
        save_shape(args.shape, inferer.shape(feature_mask, image=feature_image))
    if args.first_order is not None:
        logger.info(f"Save first-order features to: {args.first_order}")
        save_first_order(args.first_order, inferer.first_order(feature_image, feature_mask, bin_width=args.first_order_bin_width,
                                                               voxel_array_shift=args.first_order_shift))
    if args.wavelet is not None:
        logger.info(f"Save wavelet features to: {args.wavelet}")
        save_wavelet_features(args.wavelet, inferer.wavelet_features(feature_image, feature_mask, wavelet=args.wavelet_name,
                                                                     bin_width=wavelet_bin_width, classes=wavelet_classes,
                                                                     **settings))
    if args.filtered is not None:
        logger.info(f"Save filtered-image features to: {args.filtered}")
        save_filtered_features(args.filtered, inferer.filtered_features(feature_image, feature_mask, image_types=filtered_types,
                                                                        bin_width=filtered_bin_width,
                                                                        classes=filtered_classes, **settings))
    if log is not None:
        logger.info(f"Save LoG features to: {args.log}")
        save_log_features(args.log, inferer.log_features(feature_image, feature_mask, sigma=log[0], bin_width=log[1],
                                                         classes=log[2], **settings))
    if args.mesh is not None:
        logger.info(f"Save meshes to: {args.mesh}")
        os.makedirs(args.mesh, exist_ok=True)
        for m in inferer.mesh(result, image=image, space=args.mesh_space):
            if m.n_triangles or m.label == "lung":
                save_mesh(os.path.join(args.mesh, mesh_file_name(m, args.mesh_format)), m)

    if args.first_order_maps is not None:
        logger.info(f"Save first-order maps to: {args.first_order_maps}")
        save_feature_maps(args.first_order_maps,
                          inferer.first_order_maps(image, result, label=maps_label, features=maps_features,
                                                   kernel_radius=args.first_order_maps_radius,
                                                   masked_kernel=not args.first_order_maps_unmasked,
                                                   bin_width=args.first_order_bin_width,
                                                   voxel_array_shift=args.first_order_shift),
                          image, args.first_order_maps_format)

    if args.glcm_maps is not None:
        logger.info(f"Save GLCM maps to: {args.glcm_maps}")
        save_feature_maps(args.glcm_maps,
                          inferer.glcm_maps(image, result, label=glcm_label, features=glcm_features,
                                            kernel_radius=args.glcm_maps_radius, masked_kernel=not args.glcm_maps_unmasked,
                                            bin_width=args.texture_bin_width),
                          image, args.glcm_maps_format)

    if args.texture_maps is not None:
        logger.info(f"Save texture maps to: {args.texture_maps}")
        save_feature_maps(args.texture_maps,
                          inferer.texture_maps(image, result, classes=tmaps_classes, label=tmaps_label,
                                               features=tmaps_features, kernel_radius=args.texture_maps_radius,
                                               masked_kernel=not args.texture_maps_unmasked,
                                               bin_width=args.texture_bin_width),
                          image, args.texture_maps_format)


if __name__ == "__main__":
    main()
