"""The probability-map writers of lungmask_b200.io (no GPU): the 4-D NIfTI header carries the mask's spatial header
and the classes as 4th dimension, voxels in little-endian x-fastest order; unsupported targets are refused."""
import gzip
import struct

import numpy as np
import pytest


def _read(path):
    return gzip.open(path, "rb").read() if path.endswith(".gz") else open(path, "rb").read()


@pytest.mark.parametrize("ext", [".nii", ".nii.gz"])
def test_4d_nifti_header_and_byte_order(tmp_path, ext):
    from lungmask_b200 import io as lio
    K, nz, ny, nx = 3, 2, 3, 4
    probs = (np.arange(K * nz * ny * nx, dtype=np.float32) / 7.0).reshape(K, nz, ny, nx)
    D = np.zeros((3, 3))
    D[0, 0], D[2, 1], D[1, 2] = -1.0, 1.0, 1.0
    like = lio.Volume(np.zeros((nz, ny, nx), np.int16), (0.75, 1.5, 0.5), (10.0, -4.0, 2.0), tuple(D.ravel()))
    p_path, m_path = str(tmp_path / ("p" + ext)), str(tmp_path / ("m" + ext))
    lio.save_probabilities(p_path, probs, like)
    lio.save_mask(m_path, np.zeros((nz, ny, nx), np.uint8), like)
    raw, mraw = _read(p_path), _read(m_path)

    assert struct.unpack_from("<i", raw, 0)[0] == 348 and raw[344:348] == b"n+1\x00"
    assert struct.unpack_from("<8h", raw, 40)[:5] == (4, nx, ny, nz, K)
    assert struct.unpack_from("<8h", mraw, 40)[:4] == (3, nx, ny, nz)
    assert struct.unpack_from("<hh", raw, 70) == (16, 32)                          # NIFTI_TYPE_FLOAT32
    assert struct.unpack_from("<f", raw, 108)[0] == 352.0
    # the spatial header is the mask's: pixdim 1-3, qform / sform codes and the sform rows
    assert struct.unpack_from("<3f", raw, 80) == struct.unpack_from("<3f", mraw, 80)
    assert raw[252:256] == mraw[252:256] and raw[280:328] == mraw[280:328]
    srow = np.asarray([struct.unpack_from("<4f", raw, 280 + 16 * r) for r in range(3)])
    M = np.diag([-1.0, -1.0, 1.0]) @ (D * np.asarray(like.spacing))                 # LPS -> RAS, as the reader undoes
    assert np.allclose(srow[:, :3], M) and np.allclose(srow[:, 3], [-10.0, 4.0, 2.0])
    assert len(raw) == 352 + probs.nbytes
    assert raw[352:] == probs.astype("<f4").tobytes()                               # x fastest, then y, z, class
    # the 3-D reader sees the first class volume with the input geometry
    first = lio.load_input_image(p_path)
    assert np.array_equal(first.array, probs[0])
    assert np.allclose(first.GetDirection(), like.GetDirection()) and np.allclose(first.origin, like.origin)


def test_npy_and_refusals(tmp_path):
    from lungmask_b200 import io as lio
    from lungmask_b200.__main__ import build_parser
    probs = np.random.default_rng(0).random((2, 3, 4, 5), dtype=np.float32)
    lio.save_probabilities(str(tmp_path / "p.npy"), probs)
    assert np.array_equal(np.load(str(tmp_path / "p.npy")), probs)
    for bad in ("p.mha", "p.png"):
        with pytest.raises(SystemExit):
            lio.save_probabilities(str(tmp_path / bad), probs)
    with pytest.raises(ValueError):
        lio.save_probabilities(str(tmp_path / "q.npy"), probs[0])
    assert build_parser().parse_args([__file__, "o.nii", "--probabilities", "p.nii.gz"]).probabilities == "p.nii.gz"
