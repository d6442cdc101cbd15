"""Numpy restatement of the baseline JPEG encoder of csrc/jpeg.cu (include/dvc.h: dvc_encode_jpeg), stage by stage.
TEST INFRASTRUCTURE ONLY: imported by tests/ (and never by the product).

It restates libjpeg-turbo's integer arithmetic for Image.fromarray(x).save(f, "JPEG", quality=q): 4:2:0 YCbCr (jccolor.c,
jcsample.c h2v2_downsample, the edge replication of jcprepct.c), JDCT_ISLOW (jfdctint.c), the reciprocal quantizer of
jcdctmgr.c, the dummy blocks of jccoefct.c and the standard Huffman tables of jchuff.c / jstdhuff.c."""
import numpy as np

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14,
                   21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60,
                   61, 54, 47, 55, 62, 63])  # zigzag index -> natural (row-major) index

STD_LUMA_Q = [16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51, 87,
              80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101, 72, 92,
              95, 98, 112, 100, 103, 99]
STD_CHROMA_Q = [17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99, 99,
                99, 99, 99] + [99] * 32

DC_LUMA_BITS = [0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0]
DC_CHROMA_BITS = [0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0]
DC_VALS = list(range(12))
AC_LUMA_BITS = [0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7D]
AC_LUMA_VALS = [
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32, 0x81,
    0x91, 0xA1, 0x08, 0x23, 0x42, 0xB1, 0xC1, 0x15, 0x52, 0xD1, 0xF0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0A, 0x16, 0x17, 0x18,
    0x19, 0x1A, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2A, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3A, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48,
    0x49, 0x4A, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5A, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6A, 0x73, 0x74, 0x75,
    0x76, 0x77, 0x78, 0x79, 0x7A, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8A, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99,
    0x9A, 0xA2, 0xA3, 0xA4, 0xA5, 0xA6, 0xA7, 0xA8, 0xA9, 0xAA, 0xB2, 0xB3, 0xB4, 0xB5, 0xB6, 0xB7, 0xB8, 0xB9, 0xBA, 0xC2, 0xC3,
    0xC4, 0xC5, 0xC6, 0xC7, 0xC8, 0xC9, 0xCA, 0xD2, 0xD3, 0xD4, 0xD5, 0xD6, 0xD7, 0xD8, 0xD9, 0xDA, 0xE1, 0xE2, 0xE3, 0xE4, 0xE5,
    0xE6, 0xE7, 0xE8, 0xE9, 0xEA, 0xF1, 0xF2, 0xF3, 0xF4, 0xF5, 0xF6, 0xF7, 0xF8, 0xF9, 0xFA]
AC_CHROMA_BITS = [0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77]
AC_CHROMA_VALS = [
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81, 0x08,
    0x14, 0x42, 0x91, 0xA1, 0xB1, 0xC1, 0x09, 0x23, 0x33, 0x52, 0xF0, 0x15, 0x62, 0x72, 0xD1, 0x0A, 0x16, 0x24, 0x34, 0xE1, 0x25,
    0xF1, 0x17, 0x18, 0x19, 0x1A, 0x26, 0x27, 0x28, 0x29, 0x2A, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3A, 0x43, 0x44, 0x45, 0x46, 0x47,
    0x48, 0x49, 0x4A, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5A, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6A, 0x73, 0x74,
    0x75, 0x76, 0x77, 0x78, 0x79, 0x7A, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8A, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97,
    0x98, 0x99, 0x9A, 0xA2, 0xA3, 0xA4, 0xA5, 0xA6, 0xA7, 0xA8, 0xA9, 0xAA, 0xB2, 0xB3, 0xB4, 0xB5, 0xB6, 0xB7, 0xB8, 0xB9, 0xBA,
    0xC2, 0xC3, 0xC4, 0xC5, 0xC6, 0xC7, 0xC8, 0xC9, 0xCA, 0xD2, 0xD3, 0xD4, 0xD5, 0xD6, 0xD7, 0xD8, 0xD9, 0xDA, 0xE2, 0xE3, 0xE4,
    0xE5, 0xE6, 0xE7, 0xE8, 0xE9, 0xEA, 0xF2, 0xF3, 0xF4, 0xF5, 0xF6, 0xF7, 0xF8, 0xF9, 0xFA]


def huffman_codes(bits, vals):
    """(code[256], length[256]) of a canonical table (jchuff.c jpeg_make_c_derived_tbl); length 0 = no code."""
    code, length = np.zeros(256, np.int64), np.zeros(256, np.int64)
    c, k = 0, 0
    for n in range(1, 17):
        for _ in range(bits[n - 1]):
            code[vals[k]], length[vals[k]] = c, n
            c, k = c + 1, k + 1
        c <<= 1
    return code, length


DC_TABLES = (huffman_codes(DC_LUMA_BITS, DC_VALS), huffman_codes(DC_CHROMA_BITS, DC_VALS))
AC_TABLES = (huffman_codes(AC_LUMA_BITS, AC_LUMA_VALS), huffman_codes(AC_CHROMA_BITS, AC_CHROMA_VALS))


def quant_tables(q):
    """Luma and chroma tables [2,64] (natural order) of jpeg_set_quality(q, force_baseline=TRUE)."""
    q = min(max(int(q), 1), 100)
    scale = 5000 // q if q < 50 else 200 - 2 * q
    t = (np.array([STD_LUMA_Q, STD_CHROMA_Q], np.int64) * scale + 50) // 100
    return np.clip(t, 1, 255)


def ycc_planes(rgb):
    """jccolor.c rgb_ycc_convert then the padding and 4:2:0 downsampling of jcprepct.c / jcsample.c for uint8 [H,W,3]:
    Y [8 ceil(H/8), 8 ceil(W/8)] (edge replication), Cb and Cr [8 ceil(H/16), 8 ceil(W/16)] (h2v2_downsample of the
    edge-replicated full-resolution planes, rounding bias 1, 2, 1, 2 along a row; rows past the image repeat its last row)."""
    H, W, _ = rgb.shape
    x = rgb.astype(np.int64)
    R, G, B = x[..., 0], x[..., 1], x[..., 2]

    def fix(v):
        return int(v * 65536 + 0.5)

    Y = (fix(0.29900) * R + fix(0.58700) * G + fix(0.11400) * B + 32768) >> 16
    off = (128 << 16) + 32767
    Cb = (-fix(0.16874) * R - fix(0.33126) * G + fix(0.5) * B + off) >> 16
    Cr = (fix(0.5) * R - fix(0.41869) * G - fix(0.08131) * B + off) >> 16
    my, mx = -(-H // 16), -(-W // 16)
    ys, xs = np.minimum(np.arange(8 * -(-H // 8)), H - 1), np.minimum(np.arange(8 * -(-W // 8)), W - 1)
    Yp = Y[ys][:, xs]
    rows = np.minimum(np.arange(2 * -(-H // 2)), H - 1)  # the row group of an odd last row repeats it
    cols = np.minimum(np.arange(16 * mx), W - 1)
    bias = np.tile([1, 2], 4 * mx)
    nc = -(-H // 2)
    crow = np.minimum(np.arange(8 * my), nc - 1)  # chroma rows past the image repeat the last one

    def down(P):
        p = P[rows][:, cols]
        s = p[0::2, 0::2] + p[0::2, 1::2] + p[1::2, 0::2] + p[1::2, 1::2]
        return ((s + bias) >> 2)[crow]

    return Yp, down(Cb), down(Cr)


def fdct_islow(blocks):
    """jfdctint.c jpeg_fdct_islow over int64 blocks [N,8,8] of samples - 128 (output scaled by 8, as libjpeg leaves it)."""
    d = blocks.astype(np.int64).copy()
    C = {"0_298": 2446, "0_390": 3196, "0_541": 4433, "0_765": 6270, "0_899": 7373, "1_175": 9633, "1_501": 12299, "1_847": 15137,
         "1_961": 16069, "2_053": 16819, "2_562": 20995, "3_072": 25172}

    def descale(x, n):
        return (x + (1 << (n - 1))) >> n

    def one_pass(v, first):
        out = np.empty_like(v)
        tmp0, tmp7 = v[..., 0] + v[..., 7], v[..., 0] - v[..., 7]
        tmp1, tmp6 = v[..., 1] + v[..., 6], v[..., 1] - v[..., 6]
        tmp2, tmp5 = v[..., 2] + v[..., 5], v[..., 2] - v[..., 5]
        tmp3, tmp4 = v[..., 3] + v[..., 4], v[..., 3] - v[..., 4]
        tmp10, tmp13, tmp11, tmp12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
        sh = 13 - 2 if first else 13 + 2
        if first:
            out[..., 0], out[..., 4] = (tmp10 + tmp11) << 2, (tmp10 - tmp11) << 2
        else:
            out[..., 0], out[..., 4] = descale(tmp10 + tmp11, 2), descale(tmp10 - tmp11, 2)
        z1 = (tmp12 + tmp13) * C["0_541"]
        out[..., 2] = descale(z1 + tmp13 * C["0_765"], sh)
        out[..., 6] = descale(z1 - tmp12 * C["1_847"], sh)
        z1, z2, z3, z4 = tmp4 + tmp7, tmp5 + tmp6, tmp4 + tmp6, tmp5 + tmp7
        z5 = (z3 + z4) * C["1_175"]
        tmp4, tmp5, tmp6, tmp7 = tmp4 * C["0_298"], tmp5 * C["2_053"], tmp6 * C["3_072"], tmp7 * C["1_501"]
        z1, z2, z3, z4 = -z1 * C["0_899"], -z2 * C["2_562"], -z3 * C["1_961"] + z5, -z4 * C["0_390"] + z5
        out[..., 7] = descale(tmp4 + z1 + z3, sh)
        out[..., 5] = descale(tmp5 + z2 + z4, sh)
        out[..., 3] = descale(tmp6 + z2 + z3, sh)
        out[..., 1] = descale(tmp7 + z1 + z4, sh)
        return out

    d = one_pass(d, True)
    d = one_pass(d.transpose(0, 2, 1), False).transpose(0, 2, 1)
    return d


def quantize(coef, qtab):
    """jcdctmgr.c quantize with compute_reciprocal's (reciprocal, correction, shift) for divisor q << 3 (16-bit DCTELEM):
    sign(x) ((|x| + c) * recip >> r).  coef [N,64] natural order, qtab [64]."""
    out = np.empty_like(coef)
    for i in range(64):
        d = int(qtab[i]) << 3
        b = d.bit_length() - 1
        r = 16 + b
        fq, fr = (1 << r) // d, (1 << r) % d
        c = d // 2
        if fr == 0:
            fq, r = fq >> 1, r - 1
        elif fr <= d // 2:
            c += 1
        else:
            fq += 1
        a = np.abs(coef[:, i])
        v = ((a + c) * fq) >> r
        out[:, i] = np.where(coef[:, i] < 0, -v, v)
    return out


def _blocks(plane, n_by, n_bx):
    return plane[: 8 * n_by, : 8 * n_bx].reshape(n_by, 8, n_bx, 8).transpose(0, 2, 1, 3)


def quantized_blocks(rgb, q):
    """The quantized coefficients [nblocks, 64] in zigzag order and MCU order (per 16x16 MCU: Y00, Y01, Y10, Y11, Cb, Cr),
    including jccoefct.c's dummy blocks (zero AC, the DC of the preceding block of the MCU)."""
    H, W, _ = rgb.shape
    my, mx = -(-H // 16), -(-W // 16)
    Yp, Cb, Cr = ycc_planes(rgb)
    qt = quant_tables(q)
    by, bx = Yp.shape[0] // 8, Yp.shape[1] // 8

    def coded(plane, n_by, n_bx, table):
        blk = _blocks(plane - 128, n_by, n_bx).reshape(-1, 8, 8)
        return quantize(fdct_islow(blk).reshape(-1, 64), table).reshape(n_by, n_bx, 64)

    yq = coded(Yp, by, bx, qt[0])
    # the luma block grid of whole MCUs; blocks past (by, bx) are dummies
    Yq = np.zeros((2 * my, 2 * mx, 64), np.int64)
    Yq[:by, :bx] = yq
    if bx < 2 * mx:  # right dummy column: DC of the block on its left
        Yq[:by, bx, 0] = Yq[:by, bx - 1, 0]
    if by < 2 * my:  # bottom dummy row of the last MCU row: both take the DC of the MCU's block (0, 1)
        Yq[by, 0::2, 0] = Yq[by - 1, 1::2, 0]
        Yq[by, 1::2, 0] = Yq[by - 1, 1::2, 0]
    cb, cr = coded(Cb, my, mx, qt[1]), coded(Cr, my, mx, qt[1])
    Y4 = Yq.reshape(my, 2, mx, 2, 64).transpose(0, 2, 1, 3, 4).reshape(my, mx, 4, 64)
    mcu = np.concatenate([Y4, cb[:, :, None], cr[:, :, None]], axis=2).reshape(-1, 64)
    return mcu[:, ZIGZAG]


def _nbits(v):
    a = np.abs(v)
    n = np.zeros_like(a)
    while (a > 0).any():
        n += a > 0
        a >>= 1
    return n


def _events(zz):
    """Every (value, length) of the entropy-coded segment in order, per block: DC code, DC bits, per non-zero AC coefficient
    its ZRLs (runs of 16 zeros), code and bits, and EOB when the block ends in zeros.  Returns (values, lengths, block)."""
    n = zz.shape[0]
    comp = np.tile([0, 0, 0, 0, 1, 2], n // 6)
    dc = zz[:, 0]
    pred = np.zeros(n, np.int64)
    for c in range(3):
        idx = np.nonzero(comp == c)[0]
        pred[idx[1:]] = dc[idx[:-1]]
    tab = np.minimum(comp, 1)
    keys, vals, lens = [], [], []

    def add(key, v, ln):
        keys.append(key), vals.append(v), lens.append(ln)

    diff = dc - pred
    nb = _nbits(diff)
    blk = np.arange(n)
    dcode = np.where(tab == 0, DC_TABLES[0][0][nb], DC_TABLES[1][0][nb])
    dlen = np.where(tab == 0, DC_TABLES[0][1][nb], DC_TABLES[1][1][nb])
    add(blk * 1024, dcode, dlen)
    add(blk * 1024 + 1, np.where(diff < 0, diff - 1, diff) & ((1 << nb) - 1), nb)
    b, k = np.nonzero(zz[:, 1:])
    k = k + 1
    v = zz[b, k]
    first = np.ones(len(b), bool)
    first[1:] = b[1:] != b[:-1]
    prevk = np.where(first, 0, np.concatenate([[0], k[:-1]]))
    run = k - prevk - 1
    nbv = _nbits(v)
    t = tab[b]
    for j in range(3):  # at most three ZRLs before one coefficient (runs <= 62)
        m = run >= 16 * (j + 1)
        zc = np.where(t == 0, AC_TABLES[0][0][0xF0], AC_TABLES[1][0][0xF0])
        zl = np.where(t == 0, AC_TABLES[0][1][0xF0], AC_TABLES[1][1][0xF0])
        add((b * 1024 + k * 8 + j)[m], zc[m], zl[m])
    sym = ((run % 16) << 4) + nbv
    add(b * 1024 + k * 8 + 3, np.where(t == 0, AC_TABLES[0][0][sym], AC_TABLES[1][0][sym]),
        np.where(t == 0, AC_TABLES[0][1][sym], AC_TABLES[1][1][sym]))
    add(b * 1024 + k * 8 + 4, np.where(v < 0, v - 1, v) & ((1 << nbv) - 1), nbv)
    eob = zz[:, 63] == 0
    add((blk * 1024 + 1000)[eob], np.where(tab == 0, AC_TABLES[0][0][0], AC_TABLES[1][0][0])[eob],
        np.where(tab == 0, AC_TABLES[0][1][0], AC_TABLES[1][1][0])[eob])
    keys, vals, lens = (np.concatenate(a).astype(np.int64) for a in (keys, vals, lens))
    order = np.argsort(keys, kind="stable")
    return vals[order], lens[order], keys[order] // 1024


def block_bits(zz):
    """Bit length of every block's entropy-coded data [nblocks] (DC prediction per component in MCU order)."""
    _, lens, blk = _events(zz)
    return np.bincount(blk, weights=lens, minlength=zz.shape[0]).astype(np.int64)


def entropy_segment(zz):
    """The entropy-coded segment: bits packed MSB first, the last byte padded with 1-bits, 0xFF followed by 0x00."""
    vals, lens, _ = _events(zz)
    lens_nz = lens > 0
    vals, lens = vals[lens_nz], lens[lens_nz]
    total = int(lens.sum())
    start = np.concatenate([[0], np.cumsum(lens)[:-1]])
    ev = np.repeat(np.arange(len(lens)), lens)
    j = np.arange(total) - start[ev]
    bits = (vals[ev] >> (lens[ev] - 1 - j)) & 1
    pad = (-total) % 8
    bits = np.concatenate([bits, np.ones(pad, np.int64)]).astype(np.uint8)
    data = np.packbits(bits)
    ff = data == 0xFF
    out = np.repeat(data, 1 + ff)
    pos = np.cumsum(1 + ff) - 1
    out[pos[ff]] = 0
    return out.tobytes()


def header(H, W, q):
    """SOI, APP0 JFIF, DQT luma, DQT chroma, SOF0, DHT DC/AC luma, DC/AC chroma, SOS: the bytes before the scan data."""
    qt = quant_tables(q)

    def seg(marker, payload):
        return bytes([0xFF, marker]) + (len(payload) + 2).to_bytes(2, "big") + bytes(payload)

    h = bytes([0xFF, 0xD8])
    h += seg(0xE0, b"JFIF\x00" + bytes([1, 1, 0, 0, 1, 0, 1, 0, 0]))
    for t in range(2):
        h += seg(0xDB, bytes([t]) + bytes(int(v) for v in qt[t][ZIGZAG]))
    h += seg(0xC0, bytes([8]) + H.to_bytes(2, "big") + W.to_bytes(2, "big") + bytes([3, 1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1]))
    for cls_id, bits, vals in ((0x00, DC_LUMA_BITS, DC_VALS), (0x10, AC_LUMA_BITS, AC_LUMA_VALS), (0x01, DC_CHROMA_BITS, DC_VALS),
                               (0x11, AC_CHROMA_BITS, AC_CHROMA_VALS)):
        h += seg(0xC4, bytes([cls_id]) + bytes(bits) + bytes(vals))
    h += seg(0xDA, bytes([3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0]))
    return h


def encode(rgb, q=75):
    """The JFIF file of uint8 rgb [H,W,3] at quality q."""
    rgb = np.asarray(rgb, np.uint8)
    H, W, _ = rgb.shape
    return header(H, W, q) + entropy_segment(quantized_blocks(rgb, q)) + b"\xff\xd9"


KINDS = ("const", "gradient", "noise", "extreme", "stripes", "sawtooth")


def content(kind, H, W, seed=0):
    """uint8 [H,W,3] test images that reach the encoder's edge cases: a constant frame (EOB-only blocks), a smooth gradient,
    uniform noise, "extreme" 8x8 tiles of black, white and hard edges (DC differences of category 11, AC coefficients of
    category 10 at q = 100), alternate black and white rows (runs of 16+ zeros: ZRL) and a horizontal sawtooth of period 8
    (many 0xFF bytes in the entropy-coded data)."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[:H, :W]
    if kind == "const":
        return np.broadcast_to(np.array([77, 160, 23], np.uint8), (H, W, 3)).copy()
    if kind == "gradient":
        g = np.stack([x * 255 // max(W - 1, 1), y * 255 // max(H - 1, 1), (x + y) * 127 // max(H + W - 2, 1)], -1)
        return g.astype(np.uint8)
    if kind == "noise":
        return rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    if kind == "extreme":
        pick = rng.integers(0, 5, ((H + 7) // 8, (W + 7) // 8, 3))[y // 8, x // 8, :]
        yy, xx = (y % 8)[..., None], (x % 8)[..., None]
        v = np.select([pick == 0, pick == 1, pick == 2, pick == 3], [0, 255, (xx >= 4) * 255, (yy >= 4) * 255], ((xx + yy) % 2) * 255)
        return v.astype(np.uint8)
    if kind == "stripes":  # the highest vertical frequency of the DCT alone: one coefficient 34 zigzag steps after DC
        v = 128 + 100 * np.cos((2 * (y % 8) + 1) * 7 * np.pi / 16)
        return np.repeat(np.rint(v)[..., None], 3, 2).astype(np.uint8)
    if kind == "sawtooth":
        return np.stack([(x % 8) * 36, (x % 8) * 36, 255 - (x % 8) * 36], -1).astype(np.uint8)
    raise ValueError(kind)


def max_bytes(H, W):
    """include/dvc.h dvc_jpeg_max_bytes: header + EOI + twice the bytes of 1660 bits per block (DC <= 11 + 11 bits, each of
    63 AC coefficients <= 16 + 10 bits; ZRL and EOB only stand in for zero coefficients, which cost nothing else)."""
    nblk = 6 * (-(-H // 16)) * (-(-W // 16))
    return len(header(H, W, 75)) + 2 + 2 * ((1660 * nblk + 7) // 8)
