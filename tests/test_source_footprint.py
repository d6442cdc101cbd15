"""Host side of the source-resolution video output (include/dvc.h: dvc_source_footprint, dvc_ab_to_source): the footprint rule
against a brute-force enumeration in exact rationals, and the float32 oracle of the ab resampling against PyTorch's bilinear
interpolation.  No GPU needed."""
from fractions import Fraction

import numpy as np
import pytest
import torch

import source_oracle as PP

SOURCES = [(1080, 1920), (720, 1280), (480, 640), (50, 60), (481, 853), (853, 481), (37, 333), (200, 200)]
SIZES = [(432, 768), (64, 96), (80, 128)]


def _geometries():
    from dvc.prepost import centerpad_geometry

    out = []
    for Hs, Ws in SOURCES:
        for size in SIZES:
            try:
                out.append(((Hs, Ws, *centerpad_geometry(Hs, Ws, size)), size))
            except ValueError:  # the reference itself fails on this source / size
                pass
    out.append(((40, 64, 50, 80, -7, -8), (64, 96)))  # a zero-padded window larger than the resized image
    return out


GEOMETRIES = _geometries()


def _brute(geometry, size):
    """Source pixels whose centre, mapped into window coordinates, lies in [-1/2, n - 1/2] -- in exact rationals."""
    Hs, Ws, Hr, Wr, oy, ox = geometry

    def axis(n_src, n_res, off, n_win):
        inside = [i for i in range(n_src)
                  if Fraction(-1, 2) <= Fraction(2 * i + 1, 2) * Fraction(n_res, n_src) - Fraction(1, 2) - off <= Fraction(2 * n_win - 1, 2)]
        assert inside == list(range(inside[0], inside[-1] + 1))  # one contiguous run
        return inside[0], len(inside)

    y0, h = axis(Hs, Hr, oy, size[0])
    x0, w = axis(Ws, Wr, ox, size[1])
    return y0, x0, h, w


@pytest.mark.parametrize("geometry,size", GEOMETRIES)
def test_footprint_matches_exact_enumeration(geometry, size):
    import dvc

    want = _brute(geometry, size)
    assert dvc.source_footprint(*geometry, *size) == want
    assert PP.source_footprint(geometry, size) == want


def test_footprint_named_cases():
    import dvc
    from dvc.prepost import centerpad_geometry

    def fp(Hs, Ws, size=(432, 768)):
        return dvc.source_footprint(Hs, Ws, *centerpad_geometry(Hs, Ws, size), *size)

    assert fp(1080, 1920) == (0, 0, 1080, 1920)  # the window's aspect ratio: the whole frame
    assert fp(480, 640) == (60, 0, 360, 640)      # CenterPad crops: the centre band
    assert dvc.source_footprint(40, 64, 50, 80, -7, -8, 64, 96) == (0, 0, 40, 64)  # zero-padded window: the whole frame


def test_footprint_refusals():
    import dvc

    with pytest.raises(dvc.DvcError):
        dvc.source_footprint(0, 64, 50, 80, 0, 0, 64, 96)
    with pytest.raises(dvc.DvcError):  # two source rows, both centres outside the window
        dvc.source_footprint(2, 1, 1536, 768, 552, 0, 432, 768)


def _planes(seed, P, H, W):
    return np.random.default_rng(seed).standard_normal((P, H, W)).astype(np.float32) * np.float32(40)


@pytest.mark.parametrize("Hs,Ws,size", [(1080, 1920, (432, 768)), (720, 1280, (432, 768)), (100, 150, (64, 96)), (96, 64, (96, 64)),
                                        (48, 48, (80, 80))])
def test_oracle_is_bilinear_interpolation_when_uncropped(Hs, Ws, size):
    """With the resized image equal to the window (no crop, no pad) the resampling is F.interpolate(bilinear, align_corners=False)
    from the window to the source size."""
    geometry = (Hs, Ws, size[0], size[1], 0, 0)
    # PyTorch computes its source coordinates in float32 (off by up to ~3e-5 pixel at these sizes), which moves the result by
    # that fraction of a neighbour difference: smooth planes in [-1, 1], like the network's ab after its x2 bilinear up-sampling
    coarse = torch.from_numpy(np.random.default_rng(Hs + Ws).uniform(-1, 1, (1, 2, size[0] // 8, size[1] // 8)).astype(np.float32))
    ab = torch.nn.functional.interpolate(coarse, size=size, mode="bilinear", align_corners=False)[0].numpy()
    got = PP.ab_to_source(ab, geometry, size)
    want = torch.nn.functional.interpolate(torch.from_numpy(ab)[None], size=(Hs, Ws), mode="bilinear", align_corners=False)[0].numpy()
    assert got.shape == (2, Hs, Ws)
    assert np.abs(got - want).max() < 1e-4


@pytest.mark.parametrize("size", [(432, 768), (64, 96), (40, 40)])
def test_oracle_identity(size):
    ab = _planes(7, 3, *size)
    got = PP.ab_to_source(ab, (size[0], size[1], size[0], size[1], 0, 0), size)
    assert got.dtype == np.float32 and np.array_equal(got.view(np.uint32), ab.view(np.uint32))
