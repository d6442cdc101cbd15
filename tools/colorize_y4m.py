"""Colorize a YUV4MPEG2 (Y4M) stream on the device: 8-bit 4:2:0 frames in, colorized 4:2:0 frames out.

    ffmpeg -i in.mp4 -pix_fmt yuv420p -f yuv4mpegpipe - \\
      | python tools/colorize_y4m.py -i - -o - --ref exemplar.png --vgg ... --warp ... --color ... \\
      | ffmpeg -f yuv4mpegpipe -i - -colorspace bt470bg -color_range tv -c:v libx264 out.mp4

Video decoders and encoders work in planar YUV 4:2:0 (I420); this tool hands those frames to dvc_colorize_videos_i420 as they
are, so 1.5 bytes per pixel cross PCIe each way and no host core converts colour.  The conversions on the device are OpenCV's
BT.601 limited-range ones (cv2.cvtColor COLOR_YUV2RGB_I420 / COLOR_RGB2YUV_I420) with nearest-neighbour chroma; the chroma
siting tag (C420jpeg, C420mpeg2, C420paldv) is accepted and ignored.  A BT.709 source (most HD video) is therefore decoded
with the BT.601 matrix, as OpenCV decodes it, and the output is BT.601 limited range: tag it so when encoding
(-colorspace bt470bg -color_range tv), as above.

Input: progressive (no I tag, or Ip) 8-bit 4:2:0 (no C tag, C420, C420jpeg, C420mpeg2 or C420paldv) with an even width and
height.  Anything else -- C444, Cmono, C420p10, interlaced input, a bad FRAME marker, a truncated frame -- is refused.

Output: a Y4M stream with the input's F (frame rate) and A (pixel aspect) tags and its 4:2:0 tag (C420jpeg if it had none), at
--image-size, or with --source-resolution at the part of the source frame the --image-size window covers
(dvc_source_footprint; the whole frame unless CenterPad crops it).  With several --ref images, -o is a folder and exemplar
<ref>'s frames go to <folder>/<ref stem>.y4m, all colorized in one pass.

The stream goes through in chunks of --chunk frames: one dvc_colorize_videos_i420 call per chunk, each continuing from the
previous call's last_lab_out (so the frames are those of one call over the whole stream), with a reader thread filling the
next pinned input chunk and a writer thread draining the previous output chunk while the device runs.  Host and device memory
are bounded by the chunk size.  Weights and exemplars are prepared as tools/colorize_folder.py prepares them.
"""
import argparse
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "deep-exemplar-based-video-colorization_b200"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402

MAGIC = b"YUV4MPEG2"
CHROMA_420 = ("420", "420jpeg", "420mpeg2", "420paldv")  # 8-bit 4:2:0, whatever the chroma siting
MAX_LINE = 4096


class Y4MError(ValueError):
    pass


def parse_header(line):
    """The header line (with or without its newline) -> dict of the W, H (ints), F, I, A, C (strings) tags present and the list
    of X tags.  Refuses what this tool cannot colorize: a missing W / H, an odd or non-positive size, a colour format other than
    8-bit 4:2:0 and interlaced input."""
    line = line.rstrip(b"\n")
    parts = line.split(b" ")
    if parts[0] != MAGIC:
        raise Y4MError("not a YUV4MPEG2 stream (the header must start with 'YUV4MPEG2 ')")
    hdr = {"X": []}
    for p in parts[1:]:
        if not p:
            raise Y4MError("malformed header: empty tag")
        key, val = chr(p[0]), p[1:].decode("ascii", "replace")
        if key in "WH":
            if not val.isdigit() or int(val) < 1:
                raise Y4MError(f"malformed header: {key}{val}")
            hdr[key] = int(val)
        elif key in "FIAC":
            hdr[key] = val
        elif key == "X":
            hdr["X"].append(val)
        # other tags are reserved by the format and ignored
    if "W" not in hdr or "H" not in hdr:
        raise Y4MError("malformed header: W and H are required")
    if hdr.get("C", "420jpeg") not in CHROMA_420:
        raise Y4MError(f"colour format C{hdr['C']} is not supported: only 8-bit 4:2:0 (C420, C420jpeg, C420mpeg2, C420paldv); "
                       "convert with ffmpeg -pix_fmt yuv420p")
    if hdr.get("I", "p") != "p":
        raise Y4MError(f"interlaced input (I{hdr['I']}) is not supported: deinterlace first (ffmpeg -vf yadif)")
    if hdr["W"] % 2 or hdr["H"] % 2:
        raise Y4MError(f"4:2:0 frames of {hdr['W']} x {hdr['H']}: the width and the height must be even")
    return hdr


def format_header(W, H, src):
    """The output header: size W x H, progressive, the F and A tags of the input header `src` and its 4:2:0 tag (C420jpeg if it
    had none)."""
    tags = [f"W{W}", f"H{H}"]
    if "F" in src:
        tags.append(f"F{src['F']}")
    tags.append("Ip")
    if "A" in src:
        tags.append(f"A{src['A']}")
    tags.append(f"C{src.get('C', '420jpeg')}")
    return (" ".join([MAGIC.decode()] + tags) + "\n").encode()


class Y4MReader:
    """Frames of a Y4M stream (a binary file object) as I420 [3H/2, W] uint8."""

    def __init__(self, f):
        self.f = f
        line = f.readline(MAX_LINE)
        if not line:
            raise Y4MError("empty input")
        if not line.endswith(b"\n"):
            raise Y4MError("malformed header: no end of line")
        self.header = parse_header(line)
        self.W, self.H = self.header["W"], self.header["H"]
        self.frame_bytes = self.W * self.H * 3 // 2
        self.frames = 0

    def read_into(self, buf):
        """Read up to buf.shape[0] frames into the uint8 tensor buf [n, 3H/2, W]; returns how many (0 at the end)."""
        n = 0
        while n < buf.shape[0]:
            marker = self.f.readline(MAX_LINE)
            if not marker:
                break
            if not (marker == b"FRAME\n" or (marker.startswith(b"FRAME ") and marker.endswith(b"\n"))):
                raise Y4MError(f"frame {self.frames}: bad FRAME marker {marker[:32]!r}")
            view = memoryview(buf[n].numpy()).cast("B")
            got = 0
            while got < self.frame_bytes:
                k = self.f.readinto(view[got:])
                if not k:
                    raise Y4MError(f"frame {self.frames}: truncated ({got} of {self.frame_bytes} bytes)")
                got += k
            n += 1
            self.frames += 1
        return n


def write_frames(files, out, n):
    """Frames 0..n-1 of out[k] ([K, >= n, 3h/2, w] uint8, host) to files[k]."""
    for f, o in zip(files, out):
        arr = o.numpy()
        for t in range(n):
            f.write(b"FRAME\n")
            f.write(memoryview(arr[t]).cast("B"))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("-i", "--input", required=True, help="input .y4m file, or - for stdin")
    ap.add_argument("-o", "--output", required=True,
                    help="output .y4m file, or - for stdout; with several --ref, a folder that receives <ref stem>.y4m each")
    ap.add_argument("--ref", required=True, nargs="+", help="exemplar image(s), at most 8: one output stream each")
    ap.add_argument("--vgg"), ap.add_argument("--warp"), ap.add_argument("--color")
    ap.add_argument("--seeded-weights", action="store_true", help="the seeded random weights of dvc/synth.py (a smoke run only)")
    ap.add_argument("--temperature", type=float, default=1e-10)  # test.py:94
    ap.add_argument("--image-size", type=int, nargs=2, default=[216 * 2, 384 * 2], help="test.py:132")
    ap.add_argument("--wls", type=float, nargs=2, default=[500.0, 4.0], metavar=("LAMBDA", "SIGMA"),
                    help="Fast Global Smoother lambda and sigma_color (test.py:32-33); --wls 0 0 turns it off")
    ap.add_argument("--chunk", type=int, default=32, help="frames per device call (bounds device and host memory)")
    ap.add_argument("--fast", action="store_true",
                    help="one MMA per convolution product (dvc.MATH_FP16X1) instead of the fp32-class default")
    ap.add_argument("--source-resolution", action="store_true",
                    help="output at the source resolution (the part of the frame the --image-size window covers)")
    args = ap.parse_args()
    if args.chunk < 1:
        raise SystemExit("--chunk must be >= 1")
    K = len(args.ref)
    if K > 8:
        raise SystemExit("--ref: at most 8 exemplars in one pass")
    if K > 1 and args.output == "-":
        raise SystemExit("-o: with several --ref, give a folder (one stream per exemplar)")
    stems = [os.path.splitext(os.path.basename(r))[0] for r in args.ref]
    if len(set(stems)) != K:
        raise SystemExit("--ref: the exemplar file names must differ (they name the output streams)")
    H, W = args.image_size
    if H % 16 or W % 32:
        raise SystemExit("--image-size must have H % 16 == 0 and W % 32 == 0 (the networks run at half of it)")
    wls = None if args.wls == [0.0, 0.0] else tuple(args.wls)

    fin = sys.stdin.buffer if args.input == "-" else open(args.input, "rb")
    try:
        reader = Y4MReader(fin)
    except Y4MError as e:
        raise SystemExit(f"{args.input}: {e}")

    import dvc
    from colorize_folder import exemplars_lab, set_weights
    from dvc.prepost import centerpad_geometry

    Hs, Ws = reader.H, reader.W
    h, w = H, W
    if args.source_resolution:
        _, _, h, w = dvc.source_footprint(Hs, Ws, *centerpad_geometry(Hs, Ws, (H, W)), H, W)
        if h % 2 or w % 2:
            raise SystemExit(f"--source-resolution: the window covers {h} x {w} source pixels, and 4:2:0 output needs an even size")

    ctx = dvc.get_context(0)
    if args.fast:
        ctx.set_math(conv=dvc.MATH_FP16X1)
    set_weights(ctx, args.vgg, args.warp, args.color, args.seeded_weights)
    ref_lab = exemplars_lab(ctx, args.ref, (H, W))
    if K == 1:
        ctx.set_exemplar(ref_lab)
        paths = [args.output]
    else:
        ctx.set_exemplars(ref_lab)
        os.makedirs(args.output, exist_ok=True)
        paths = [os.path.join(args.output, s + ".y4m") for s in stems]
    files = [sys.stdout.buffer if p == "-" else open(p, "wb") for p in paths]
    head = format_header(w, h, reader.header)
    for f in files:
        f.write(head)

    C = args.chunk
    ring_in = [torch.empty(C, Hs * 3 // 2, Ws, dtype=torch.uint8).pin_memory() for _ in range(2)]
    ring_out = [None, None]
    writes = [None, None]
    io_in, io_out = ThreadPoolExecutor(1), ThreadPoolExecutor(1)
    t0 = time.perf_counter()
    pending = io_in.submit(reader.read_into, ring_in[0])
    last, i, total = None, 0, 0
    try:
        while True:
            try:
                n = pending.result()
            except Y4MError as e:
                raise SystemExit(f"{args.input}: {e}")
            if n == 0:
                break
            slot = i & 1
            pending = io_in.submit(reader.read_into, ring_in[slot ^ 1])  # the previous call is done with that chunk
            if writes[slot] is not None:  # the writes of chunk i-2 still read this output slot
                writes[slot].result()
            if ring_out[slot] is None or ring_out[slot].shape[1] != n:
                ring_out[slot] = torch.empty(K, n, h * 3 // 2, w, dtype=torch.uint8).pin_memory()
            out, last = ctx.colorize_videos_i420([ring_in[slot][:n]], [K], (H, W), args.temperature, first_last_lab=last, wls=wls,
                                                 source_resolution=args.source_resolution, out_format="i420",
                                                 out=[ring_out[slot]], return_last=True)
            writes[slot] = io_out.submit(write_frames, files, out[0], n)
            total += n
            i += 1
        for wr in writes:
            if wr is not None:
                wr.result()
    finally:
        io_in.shutdown(), io_out.shutdown()
        for f in files:
            f.flush()
            if f is not sys.stdout.buffer:
                f.close()
    dt = time.perf_counter() - t0
    for p in paths:
        print(f"{total} frames -> {p if p != '-' else 'stdout'}", file=sys.stderr)
    print(f"streamed {total} frames in {dt:.3f} s ({total / dt:.1f} frames/s after start-up)", file=sys.stderr)


if __name__ == "__main__":
    main()
