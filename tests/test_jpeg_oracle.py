"""The numpy JPEG encoder of tests/jpeg_oracle.py against Pillow (libjpeg-turbo), byte for byte.  CPU only: it pins the
arithmetic that csrc/jpeg.cu restates, so the GPU tests can compare the device encoder with either."""
import io

import numpy as np
import pytest

import jpeg_oracle as J

PIL = pytest.importorskip("PIL")
from PIL import Image, features  # noqa: E402

pytestmark = pytest.mark.skipif(not features.check_feature("libjpeg_turbo"),
                                reason="Pillow is not built against libjpeg-turbo, whose arithmetic the encoder restates")

QUALITIES = (1, 10, 50, 75, 95, 100)
# every residue class of H mod 16 and of W mod 16, and the named sizes (a 1x1 image, odd sizes, a cropped footprint, the
# window and 1080p)
RESIDUE_SIZES = [(16 + r, 16 + (7 * r + 5) % 16) for r in range(16)]
SMALL_SIZES = [(1, 1), (7, 9), (8, 8), (17, 33)] + RESIDUE_SIZES
LARGE_SIZES = [(360, 640), (432, 768), (1080, 1920)]


def pillow_jpeg(rgb, q):
    buf = io.BytesIO()
    Image.fromarray(np.ascontiguousarray(rgb)).save(buf, "JPEG", quality=q)
    return buf.getvalue()


def test_residue_classes_covered():
    assert {h % 16 for h, _ in RESIDUE_SIZES} == set(range(16)) and {w % 16 for _, w in RESIDUE_SIZES} == set(range(16))


@pytest.mark.parametrize("kind", J.KINDS)
@pytest.mark.parametrize("hw", SMALL_SIZES, ids=lambda hw: f"{hw[0]}x{hw[1]}")
def test_small_sizes_equal_pillow(hw, kind):
    img = J.content(kind, *hw, seed=hw[0] * 1000 + hw[1])
    for q in QUALITIES:
        got = J.encode(img, q)
        assert got == pillow_jpeg(img, q), (hw, kind, q)
        assert len(got) <= J.max_bytes(*hw)


@pytest.mark.parametrize("hw", LARGE_SIZES, ids=lambda hw: f"{hw[0]}x{hw[1]}")
def test_large_sizes_equal_pillow(hw):
    # every quality once, each with another kind of content (the full matrix at 1080p takes minutes in numpy)
    for q, kind in zip(QUALITIES, ("gradient", "noise", "extreme", "stripes", "sawtooth", "const")):
        img = J.content(kind, *hw, seed=q)
        got = J.encode(img, q)
        assert got == pillow_jpeg(img, q), (hw, kind, q)
        assert len(got) <= J.max_bytes(*hw)


def test_header_is_pillows():
    for (H, W), q in (((1, 1), 1), ((1080, 1920), 75), ((17, 33), 100)):
        img = J.content("gradient", H, W)
        assert pillow_jpeg(img, q).startswith(J.header(H, W, q))


def test_content_reaches_the_edge_cases():
    """The matrix exercises DC differences of category 11, AC values of category 10, ZRL runs, EOB-only blocks and 0xFF
    stuffing -- checked on the oracle's intermediate stages, so a change of the content generator cannot lose them."""
    def stats(kind, q):
        zz = J.quantized_blocks(J.content(kind, 64, 96), q)
        comp = np.tile([0, 0, 0, 0, 1, 2], len(zz) // 6)
        dc = max(int(np.abs(np.diff(zz[comp == c, 0])).max(initial=0)) for c in range(3))
        run = 0
        for row in zz:
            nz = np.nonzero(row[1:])[0] + 1
            if len(nz):
                run = max(run, int(np.diff(np.concatenate([[0], nz])).max()) - 1)
        seg = J.entropy_segment(zz)
        return dc, int(np.abs(zz[:, 1:]).max()), run, seg.count(b"\xff\x00"), bool((zz[:, 1:] == 0).all(axis=1).all())

    assert stats("extreme", 100)[0] >= 1024 and stats("extreme", 100)[1] >= 512  # DC category 11, AC category 10
    assert stats("stripes", 75)[2] >= 32  # two ZRLs before one coefficient
    assert stats("sawtooth", 100)[3] >= 64  # stuffed bytes
    assert stats("const", 75)[4]  # every block is DC + EOB


def test_library_bound_is_the_oracles():
    """dvc_jpeg_max_bytes needs no device: the library's bound is the oracle's, and sizes outside the encoder's are refused."""
    import dvc

    for hw in SMALL_SIZES + LARGE_SIZES + [(65535, 1), (2160, 3840)]:
        assert dvc.jpeg_max_bytes(*hw) == J.max_bytes(*hw), hw
    for hw in ((0, 5), (5, 0), (65536, 8), (8192, 8192)):
        with pytest.raises(dvc.DvcError):
            dvc.jpeg_max_bytes(*hw)


def test_stage_shapes():
    img = J.content("noise", 17, 33)
    Y, Cb, Cr = J.ycc_planes(img)
    assert Y.shape == (24, 40) and Cb.shape == Cr.shape == (16, 24)
    zz = J.quantized_blocks(img, 75)
    assert zz.shape == (6 * 2 * 3, 64)
    bits = J.block_bits(zz)
    assert len(J.entropy_segment(zz)) >= (int(bits.sum()) + 7) // 8
