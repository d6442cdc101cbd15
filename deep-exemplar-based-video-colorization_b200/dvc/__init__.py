"""ctypes binding of libdvc.so (include/dvc.h) -- the only way Python reaches the CUDA kernels.

PyTorch is used for device memory, streams and torch.distributed; every FLOP of the hot path runs
in hand-written sm_90a kernels inside libdvc.so.  There is no CPU fallback and no torch fallback:
if the library or a CUDA device is missing, every entry point raises.
"""
import ctypes
import os
import threading

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(os.path.dirname(_HERE), "lib", "libdvc.so")

NET_VGG, NET_WARP, NET_COLOR = 0, 1, 2
MATH_FP32, MATH_TF32X3, MATH_BF16X3, MATH_FP16X3 = 0, 1, 2, 3
# convolutions only, opt-in: one MMA per product on the operand planes' hi parts (11-bit operands, the precision of
# PyTorch's cuDNN convolutions with TF32 allowed); see include/dvc.h
MATH_FP16X1 = 4

EXPORTED = [
    "dvc_create", "dvc_destroy", "dvc_last_error", "dvc_version", "dvc_set_math", "dvc_set_weight",
    "dvc_vgg19_forward", "dvc_warpnet_forward", "dvc_colorvidnet_forward", "dvc_corr_softmax_warp",
    "dvc_set_exemplar", "dvc_colorize_frames", "dvc_colorize_clip", "dvc_exemplar_pack_size",
    "dvc_exemplar_export", "dvc_exemplar_import", "dvc_launch_count", "dvc_profile_corr", "dvc_corr_mean_ms",
    "dvc_debug_set_flag", "dvc_debug_get_buffer", "dvc_debug_conv2d", "dvc_profile_conv", "dvc_conv_profile",
    "dvc_resize_half", "dvc_upsample2_scaled", "dvc_lab_to_rgb8", "dvc_rgb8_to_lab",
    "dvc_fgs_filter", "dvc_l_to_guide8", "dvc_resize_antialias_crop_rgb8", "dvc_contextual_loss_forward",
    "dvc_peer_buffer_create", "dvc_peer_buffer_open", "dvc_peer_buffer_close", "dvc_peer_buffer_destroy",
    "dvc_corr_set_peer_outputs", "dvc_set_exemplars", "dvc_colorize_frames_exemplars", "dvc_colorize_clip_exemplars",
    "dvc_corr_softmax_warp_exemplars", "dvc_colorize_video_rgb8", "dvc_colorize_frames_clips", "dvc_colorize_clips",
    "dvc_colorize_videos_rgb8", "dvc_colorize_frames_clips_exemplars", "dvc_colorize_clips_exemplars",
    "dvc_colorize_videos_exemplars_rgb8", "dvc_source_footprint", "dvc_ab_to_source", "dvc_colorize_videos_source_rgb8",
    "dvc_jpeg_max_bytes", "dvc_encode_jpeg", "dvc_colorize_videos_jpeg", "dvc_colorize_videos_gray8",
    "dvc_i420_to_rgb8", "dvc_rgb8_to_i420", "dvc_colorize_videos_i420", "dvc_debug_resize_taps",
]

_lib = None
_lib_lock = threading.Lock()


class DvcError(RuntimeError):
    pass


def load_library():
    """dlopen libdvc.so and declare the prototypes of include/dvc.h.  Fails loudly if it is not built."""
    global _lib
    with _lib_lock:
        if _lib is not None:
            return _lib
        if not os.path.isfile(LIB_PATH):
            raise DvcError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no fallback implementation)")
        lib = ctypes.CDLL(LIB_PATH)
        c_void, c_int, c_float, c_i64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_int64
        P = ctypes.POINTER
        lib.dvc_create.argtypes = [P(c_void), c_int]
        lib.dvc_destroy.argtypes = [c_void]
        lib.dvc_last_error.argtypes = [c_void]
        lib.dvc_last_error.restype = ctypes.c_char_p
        lib.dvc_version.restype = ctypes.c_char_p
        lib.dvc_set_math.argtypes = [c_void, c_int, c_int]
        lib.dvc_set_weight.argtypes = [c_void, c_int, ctypes.c_char_p, c_void, P(c_i64), c_int]
        lib.dvc_vgg19_forward.argtypes = [c_void, c_void, c_int, c_int, c_int, c_int, P(ctypes.c_char_p), P(c_void),
                                          c_int, c_void]
        lib.dvc_warpnet_forward.argtypes = [c_void, c_void, P(c_void), P(c_void), c_int, c_int, c_int, c_float, c_float,
                                            c_int, c_void, c_void, c_void]
        lib.dvc_colorvidnet_forward.argtypes = [c_void, c_void, c_int, c_int, c_int, c_void, c_void]
        lib.dvc_corr_softmax_warp.argtypes = [c_void, c_void, c_void, c_void, c_int, c_int, c_int, c_int, c_int, c_float,
                                              c_void, c_void, c_void, c_void]
        lib.dvc_set_exemplar.argtypes = [c_void, c_void, c_int, c_int, c_void]
        lib.dvc_colorize_frames.argtypes = [c_void, c_void, c_void, c_int, c_int, c_int, c_float, c_void, c_void, c_void,
                                            c_void]
        lib.dvc_colorize_clip.argtypes = [c_void, c_void, c_int, c_int, c_int, c_float, c_void, c_void, c_void]
        lib.dvc_set_exemplars.argtypes = [c_void, c_void, c_int, c_int, c_int, c_void]
        lib.dvc_colorize_frames_exemplars.argtypes = [c_void, c_void, c_void, c_int, c_int, c_int, c_float, c_void, c_void,
                                                      c_void, c_void]
        lib.dvc_colorize_clip_exemplars.argtypes = [c_void, c_void, c_int, c_int, c_int, c_float, c_void, c_int, c_void, c_void]
        lib.dvc_corr_softmax_warp_exemplars.argtypes = [c_void, c_void, c_void, c_void, c_int, c_int, c_int, c_int, c_float,
                                                        c_void, c_void, c_void, c_void]
        lib.dvc_colorize_video_rgb8.argtypes = [c_void, c_void, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                                                c_float, c_void, c_int, c_float, c_float, c_void, c_void, c_void]
        lib.dvc_colorize_frames_clips.argtypes = [c_void, c_void, c_void, c_int, c_int, c_int, c_float, c_void, c_void, c_void,
                                                  c_void]
        lib.dvc_colorize_clips.argtypes = [c_void, c_void, c_int, c_int, c_int, c_float, c_void, c_int, c_void, c_void]
        lib.dvc_colorize_videos_rgb8.argtypes = [c_void, c_int, P(c_void), c_int, P(c_int), c_int, c_int, c_float, c_void, c_int,
                                                 c_float, c_float, c_void, c_void, c_void]
        lib.dvc_colorize_frames_clips_exemplars.argtypes = [c_void, c_void, c_void, c_int, P(c_int), c_int, c_int, c_float, c_void,
                                                            c_void, c_void, c_void]
        lib.dvc_colorize_clips_exemplars.argtypes = [c_void, c_void, c_int, c_int, c_int, c_float, c_void, c_int, P(c_int), c_void,
                                                     c_void]
        lib.dvc_colorize_videos_exemplars_rgb8.argtypes = [c_void, c_int, P(c_int), P(c_void), c_int, P(c_int), c_int, c_int, c_float,
                                                           c_void, c_int, c_float, c_float, c_void, c_void, c_void]
        lib.dvc_source_footprint.argtypes = [c_int] * 8 + [P(c_int)]
        lib.dvc_ab_to_source.argtypes = [c_void, c_void] + [c_int] * 9 + [c_void, c_void]
        lib.dvc_colorize_videos_source_rgb8.argtypes = [c_void, c_int, P(c_int), P(c_void), c_int, P(c_int), c_int, c_int, c_float,
                                                        c_void, c_int, c_float, c_float, P(c_void), c_void, c_void]
        lib.dvc_jpeg_max_bytes.argtypes = [c_int, c_int]
        lib.dvc_jpeg_max_bytes.restype = c_i64
        lib.dvc_encode_jpeg.argtypes = [c_void, c_void, c_int, c_int, c_int, c_int, c_void, c_i64, c_void, c_void]
        lib.dvc_colorize_videos_jpeg.argtypes = [c_void, c_int, P(c_int), P(c_void), c_int, P(c_int), c_int, c_int, c_float, c_void,
                                                 c_int, c_float, c_float, c_int, c_int, P(c_void), c_i64, c_void, c_void, c_void]
        lib.dvc_colorize_videos_gray8.argtypes = lib.dvc_colorize_videos_jpeg.argtypes
        lib.dvc_i420_to_rgb8.argtypes = [c_void, c_void, c_int, c_int, c_int, c_void, c_void]
        lib.dvc_rgb8_to_i420.argtypes = [c_void, c_void, c_int, c_int, c_int, c_void, c_void]
        lib.dvc_colorize_videos_i420.argtypes = [c_void, c_int, P(c_int), P(c_void), c_int, P(c_int), c_int, c_int, c_float, c_void,
                                                 c_int, c_float, c_float, c_int, c_int, P(c_void), c_void, c_void]
        lib.dvc_exemplar_pack_size.argtypes = [c_void, c_int, c_int]
        lib.dvc_exemplar_pack_size.restype = c_i64
        lib.dvc_exemplar_export.argtypes = [c_void, c_void, c_i64, c_void]
        lib.dvc_exemplar_import.argtypes = [c_void, c_void, c_i64, c_int, c_int, c_void]
        lib.dvc_launch_count.argtypes = [c_void, c_int]
        lib.dvc_launch_count.restype = c_i64
        lib.dvc_profile_corr.argtypes = [c_void, c_int]
        lib.dvc_corr_mean_ms.argtypes = [c_void, c_int]
        lib.dvc_corr_mean_ms.restype = ctypes.c_double
        lib.dvc_resize_half.argtypes = [c_void, c_void, c_int, c_int, c_int, c_void, c_void]
        lib.dvc_upsample2_scaled.argtypes = [c_void, c_void, c_int, c_int, c_int, c_float, c_void, c_void]
        lib.dvc_lab_to_rgb8.argtypes = [c_void, c_void, c_void, c_int, c_int, c_int, c_void, c_void]
        lib.dvc_rgb8_to_lab.argtypes = [c_void, c_void, c_int, c_int, c_int, c_void, c_void]
        lib.dvc_fgs_filter.argtypes = [c_void, c_void, c_void, c_int, c_int, c_int, c_float, c_float, c_float, c_int, c_void, c_void]
        lib.dvc_l_to_guide8.argtypes = [c_void, c_void, c_int, c_int, c_void, c_void]
        lib.dvc_resize_antialias_crop_rgb8.argtypes = [c_void, c_void, c_int, c_int, c_int, c_int, c_int, c_int, c_void, c_int, c_int,
                                                       c_void]
        lib.dvc_contextual_loss_forward.argtypes = [c_void, c_void, c_void, c_int, c_int, c_int, c_int, c_float, c_int, c_void, c_void]
        lib.dvc_peer_buffer_create.argtypes = [c_void, c_i64, P(c_void), ctypes.c_char_p]
        lib.dvc_peer_buffer_open.argtypes = [c_void, ctypes.c_char_p, P(c_void)]
        lib.dvc_peer_buffer_close.argtypes = [c_void, c_void]
        lib.dvc_peer_buffer_destroy.argtypes = [c_void, c_void]
        lib.dvc_corr_set_peer_outputs.argtypes = [c_void, c_int, P(c_void), P(c_void), c_i64]
        lib.dvc_profile_conv.argtypes = [c_void, c_int]
        lib.dvc_conv_profile.argtypes = [c_void, c_int, c_int, P(ctypes.c_double), P(ctypes.c_double)]
        lib.dvc_debug_set_flag.argtypes = [c_void, ctypes.c_char_p, c_int]
        lib.dvc_debug_get_buffer.argtypes = [c_void, ctypes.c_char_p, P(c_void), P(c_i64), P(c_int)]
        lib.dvc_debug_conv2d.argtypes = [c_void, c_int, ctypes.c_char_p, c_void, c_int, c_int, c_int, c_int, c_int, c_int, c_float,
                                         c_int, c_int, c_int, c_float, c_int, c_void, c_void, c_void, c_void]
        lib.dvc_debug_resize_taps.argtypes = [c_int, c_int, P(ctypes.c_double), c_int, P(c_int)]
        _lib = lib
        return lib


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _stream(device):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _dev_f32(t, what):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise DvcError(f"{what}: expected a CUDA tensor (libdvc has no CPU path)")
    if t.dtype != torch.float32:
        raise DvcError(f"{what}: expected float32, got {t.dtype}")
    return t.contiguous()


class Context:
    """One dvc_ctx per CUDA device; owns the weights of all three networks and all workspaces."""

    def __init__(self, device=0):
        self.lib = load_library()
        if not torch.cuda.is_available():
            raise DvcError("no CUDA device visible: libdvc has no CPU fallback")
        self.device = torch.device("cuda", device if isinstance(device, int) else torch.device(device).index or 0)
        h = ctypes.c_void_p(0)
        rc = self.lib.dvc_create(ctypes.byref(h), self.device.index)
        if rc != 0:
            raise DvcError(f"dvc_create failed ({rc}): {self.lib.dvc_last_error(None).decode()}")
        self.h = h
        self._weight_sig = {}
        self.n_exemplars = 1  # exemplars cached by set_exemplar(s) / exemplar_import (sizes the *_exemplars outputs)

    def close(self):
        if getattr(self, "h", None):
            self.lib.dvc_destroy(self.h)
            self.h = None

    def _check(self, rc, what):
        if rc != 0:
            raise DvcError(f"{what} failed ({rc}): {self.lib.dvc_last_error(self.h).decode()}")

    # ---- configuration / weights -------------------------------------------------------------
    def set_math(self, conv=MATH_TF32X3, corr=MATH_FP16X3):
        self._check(self.lib.dvc_set_math(self.h, conv, corr), "dvc_set_math")

    def set_weights(self, net, state_dict):
        """Replaces load_state_dict (test.py:150,158-159) for `net` in {NET_VGG, NET_WARP, NET_COLOR}."""
        self._weight_sig.pop(net, None)  # a drop-in module that synced earlier must re-upload on its next forward
        for key, t in state_dict.items():
            t = t.detach().to(torch.float32).contiguous()
            shape = (ctypes.c_int64 * t.dim())(*t.shape)
            self._check(self.lib.dvc_set_weight(self.h, net, key.encode(), _ptr(t), shape, t.dim()),
                        f"dvc_set_weight({key})")

    def sync_module_weights(self, net, module):
        """Push a drop-in module's parameters when they changed (load_state_dict / .cuda() / in-place edit)."""
        sd = module.state_dict()
        sig = tuple((k, v.data_ptr(), v._version, tuple(v.shape)) for k, v in sd.items())
        if self._weight_sig.get(net) != sig:
            self.set_weights(net, sd)
            self._weight_sig[net] = sig

    # ---- module-level drop-ins -----------------------------------------------------------------
    def vgg19_forward(self, x, out_keys, preprocess=True):
        x = _dev_f32(x, "VGG19 input")
        if x.dim() != 4 or x.shape[1] != 3:
            raise DvcError("VGG19 input must be [B,3,H,W]")
        B, _, H, W = x.shape
        dims = {}
        h, w = H, W
        chans = [64, 128, 256, 512, 512]
        nconv = [2, 2, 4, 4, 4]
        for blk in range(5):
            for i in range(nconv[blk]):
                dims[f"r{blk + 1}{i + 1}"] = (chans[blk], h, w)
            h, w = h // 2, w // 2
            dims[f"p{blk + 1}"] = (chans[blk], h, w)
        outs = []
        for k in out_keys:
            if k not in dims:
                raise DvcError(f"unknown VGG key {k!r}")
            c, hh, ww = dims[k]
            outs.append(torch.empty(B, c, hh, ww, device=x.device, dtype=torch.float32))
        keys = (ctypes.c_char_p * len(out_keys))(*[k.encode() for k in out_keys])
        ptrs = (ctypes.c_void_p * len(outs))(*[o.data_ptr() for o in outs])
        rc = self.lib.dvc_vgg19_forward(self.h, _ptr(x), B, H, W, 1 if preprocess else 0, keys, ptrs, len(outs),
                                        _stream(x.device))
        self._check(rc, "dvc_vgg19_forward")
        return outs

    def warpnet_forward(self, B_lab_map, A_feats, B_feats, temperature, wta_scale_weight=1.0, reuse_exemplar=False):
        B_lab_map = _dev_f32(B_lab_map, "B_lab_map")
        A = [_dev_f32(t, "A feature") for t in A_feats]
        Bf = [_dev_f32(t, "B feature") for t in B_feats]
        Bn, ch, H, W = B_lab_map.shape
        if ch != 3:
            raise DvcError("B_lab_map must have 3 channels")
        y = torch.empty(Bn, 3, H, W, device=B_lab_map.device, dtype=torch.float32)
        sim = torch.empty(Bn, 1, H, W, device=B_lab_map.device, dtype=torch.float32)
        pa = (ctypes.c_void_p * 4)(*[t.data_ptr() for t in A])
        pb = (ctypes.c_void_p * 4)(*[t.data_ptr() for t in Bf])
        rc = self.lib.dvc_warpnet_forward(self.h, _ptr(B_lab_map), pa, pb, Bn, H, W, float(temperature),
                                          float(wta_scale_weight), 1 if reuse_exemplar else 0, _ptr(y), _ptr(sim),
                                          _stream(B_lab_map.device))
        self._check(rc, "dvc_warpnet_forward")
        return y, sim

    def colorvidnet_forward(self, x):
        x = _dev_f32(x, "ColorVidNet input")
        if x.dim() != 4 or x.shape[1] != 7:
            raise DvcError("ColorVidNet input must be [B,7,H,W]")
        B, _, H, W = x.shape
        out = torch.empty(B, 2, H, W, device=x.device, dtype=torch.float32)
        self._check(self.lib.dvc_colorvidnet_forward(self.h, _ptr(x), B, H, W, _ptr(out), _stream(x.device)),
                    "dvc_colorvidnet_forward")
        return out

    def corr_softmax_warp(self, theta_hat, phi_hat, V, temperature, want_argmax=False):
        """theta_hat [B,C,NA], phi_hat [Bphi,C,NB], V [Bphi,NB,3] -> y [B,NA,3], sim [B,NA] (, argmax)."""
        theta_hat, phi_hat, V = _dev_f32(theta_hat, "theta_hat"), _dev_f32(phi_hat, "phi_hat"), _dev_f32(V, "V")
        B, C, NA = theta_hat.shape
        Bphi, _, NB = phi_hat.shape
        y = torch.empty(B, NA, 3, device=theta_hat.device, dtype=torch.float32)
        sim = torch.empty(B, NA, device=theta_hat.device, dtype=torch.float32)
        am = torch.empty(B, NA, device=theta_hat.device, dtype=torch.int32) if want_argmax else None
        rc = self.lib.dvc_corr_softmax_warp(self.h, _ptr(theta_hat), _ptr(phi_hat), _ptr(V), B, Bphi, NA, NB, C,
                                            float(temperature), _ptr(y), _ptr(sim), _ptr(am), _stream(theta_hat.device))
        self._check(rc, "dvc_corr_softmax_warp")
        return (y, sim, am) if want_argmax else (y, sim)

    def corr_softmax_warp_exemplars(self, theta_hat, phi_hat, V, temperature, want_argmax=False):
        """One query set theta_hat [1,C,NA] against K reference sets phi_hat [K,C,NB], V [K,NB,3] -> y [K,NA,3],
        sim [K,NA] (, argmax [K,NA])."""
        theta_hat, phi_hat, V = _dev_f32(theta_hat, "theta_hat"), _dev_f32(phi_hat, "phi_hat"), _dev_f32(V, "V")
        _, C, NA = theta_hat.shape
        K, _, NB = phi_hat.shape
        if theta_hat.shape[0] != 1 or phi_hat.shape[1] != C or tuple(V.shape) != (K, NB, 3):
            raise DvcError("corr_softmax_warp_exemplars: expected theta_hat [1,C,NA], phi_hat [K,C,NB], V [K,NB,3]")
        y = torch.empty(K, NA, 3, device=theta_hat.device, dtype=torch.float32)
        sim = torch.empty(K, NA, device=theta_hat.device, dtype=torch.float32)
        am = torch.empty(K, NA, device=theta_hat.device, dtype=torch.int32) if want_argmax else None
        rc = self.lib.dvc_corr_softmax_warp_exemplars(self.h, _ptr(theta_hat), _ptr(phi_hat), _ptr(V), K, NA, NB, C,
                                                      float(temperature), _ptr(y), _ptr(sim), _ptr(am), _stream(theta_hat.device))
        self._check(rc, "dvc_corr_softmax_warp_exemplars")
        return (y, sim, am) if want_argmax else (y, sim)

    # ---- fused per-frame / per-clip path ---------------------------------------------------------
    def set_exemplar(self, IB_lab):
        t = IB_lab.detach().to(torch.float32).contiguous()
        if t.dim() != 4 or t.shape[0] != 1 or t.shape[1] != 3:
            raise DvcError("exemplar must be [1,3,H,W]")
        self._check(self.lib.dvc_set_exemplar(self.h, _ptr(t), t.shape[2], t.shape[3], _stream(self.device)),
                    "dvc_set_exemplar")
        self.n_exemplars = 1
        if not t.is_cuda:
            torch.cuda.current_stream(self.device).synchronize()  # the host buffer must outlive the async copy

    def set_exemplars(self, IB_lab):
        """K exemplars [K,3,H,W] (test.py:168-181 runs the clip once per reference image): each gets set_exemplar's
        prologue into a slot of its own; colorize_frames_exemplars / colorize_clip_exemplars then run against all K."""
        t = IB_lab.detach().to(torch.float32).contiguous()
        if t.dim() != 4 or t.shape[1] != 3:
            raise DvcError("exemplars must be [K,3,H,W]")
        self._check(self.lib.dvc_set_exemplars(self.h, _ptr(t), t.shape[0], t.shape[2], t.shape[3], _stream(self.device)),
                    "dvc_set_exemplars")
        self.n_exemplars = t.shape[0]
        if not t.is_cuda:
            torch.cuda.current_stream(self.device).synchronize()

    def colorize_frames_exemplars(self, IA_l, last, temperature=1e-10, want_warp=False):
        """One frame IA_l [1,1,H,W] against the K cached exemplars, last [K,3,H,W] -> ab [K,2,H,W]
        (, warp [K,3,H,W], sim [K,1,H,W])."""
        IA_l, last = _dev_f32(IA_l, "IA_l"), _dev_f32(last, "last")
        _, c1, H, W = IA_l.shape
        K = last.shape[0]
        if IA_l.shape[0] != 1 or c1 != 1 or tuple(last.shape[1:]) != (3, H, W):
            raise DvcError("colorize_frames_exemplars: IA_l must be [1,1,H,W] and last [K,3,H,W]")
        ab = torch.empty(K, 2, H, W, device=IA_l.device, dtype=torch.float32)
        warp = torch.empty(K, 3, H, W, device=IA_l.device, dtype=torch.float32) if want_warp else None
        sim = torch.empty(K, 1, H, W, device=IA_l.device, dtype=torch.float32) if want_warp else None
        rc = self.lib.dvc_colorize_frames_exemplars(self.h, _ptr(IA_l), _ptr(last), K, H, W, float(temperature), _ptr(ab),
                                                    _ptr(warp), _ptr(sim), _stream(IA_l.device))
        self._check(rc, "dvc_colorize_frames_exemplars")
        return (ab, warp, sim) if want_warp else ab

    def colorize_clip_exemplars(self, L, temperature=1e-10, first_last_lab=None, out=None):
        """L [F,1,H,W] -> ab [K,F,2,H,W]: colorize_clip against each of the K cached exemplars (K independent recurrences,
        test.py:76-96), with the exemplar-independent half of every frame computed once.  first_last_lab: None (zeros) or
        [K,3,H,W].  L pinned on the host or on the device; `out` lives where L lives."""
        if L.dtype != torch.float32 or L.dim() != 4 or L.shape[1] != 1:
            raise DvcError("colorize_clip_exemplars takes a float32 [F,1,H,W] tensor")
        L = L.contiguous()
        F_, _, H, W = L.shape
        K = self.n_exemplars
        if out is None:
            out = torch.empty(K, F_, 2, H, W, dtype=torch.float32, device=L.device)
            if not L.is_cuda:
                out = out.pin_memory()
        if out.is_cuda != L.is_cuda or not out.is_contiguous() or tuple(out.shape) != (K, F_, 2, H, W):
            raise DvcError("colorize_clip_exemplars: `out` must be a contiguous [K,F,2,H,W] tensor on the same side as L")
        fl = None
        if first_last_lab is not None:
            fl = first_last_lab.to(torch.float32).contiguous()
            if tuple(fl.shape) != (K, 3, H, W):
                raise DvcError("colorize_clip_exemplars: first_last_lab must be [K,3,H,W]")
        rc = self.lib.dvc_colorize_clip_exemplars(self.h, _ptr(L), F_, H, W, float(temperature), _ptr(fl), K, _ptr(out),
                                                  _stream(self.device))
        self._check(rc, "dvc_colorize_clip_exemplars")
        return out

    def colorize_frames(self, IA_l, IA_last_lab, temperature=1e-10, want_warp=False):
        IA_l, IA_last_lab = _dev_f32(IA_l, "IA_l"), _dev_f32(IA_last_lab, "IA_last_lab")
        B, c1, H, W = IA_l.shape
        if c1 != 1 or tuple(IA_last_lab.shape) != (B, 3, H, W):
            raise DvcError("IA_l must be [B,1,H,W] and IA_last_lab [B,3,H,W]")
        ab = torch.empty(B, 2, H, W, device=IA_l.device, dtype=torch.float32)
        warp = torch.empty(B, 3, H, W, device=IA_l.device, dtype=torch.float32) if want_warp else None
        sim = torch.empty(B, 1, H, W, device=IA_l.device, dtype=torch.float32) if want_warp else None
        rc = self.lib.dvc_colorize_frames(self.h, _ptr(IA_l), _ptr(IA_last_lab), B, H, W, float(temperature), _ptr(ab),
                                          _ptr(warp), _ptr(sim), _stream(IA_l.device))
        self._check(rc, "dvc_colorize_frames")
        return (ab, warp, sim) if want_warp else ab

    def colorize_clip(self, L, temperature=1e-10, first_last_lab=None, out=None):
        """L [F,1,H,W] -> ab [F,2,H,W] with the recurrence of test.py:76-96 kept on the device.

        L may be a pinned CPU tensor (one host->device copy of L and one device->host copy of ab per frame inside
        the call) or a CUDA tensor (frames already resident in HBM); `out` lives where L lives."""
        if L.dtype != torch.float32 or L.dim() != 4 or L.shape[1] != 1:
            raise DvcError("colorize_clip takes a float32 [F,1,H,W] tensor")
        L = L.contiguous()
        F_, _, H, W = L.shape
        if out is None:
            out = torch.empty(F_, 2, H, W, dtype=torch.float32, device=L.device)
            if not L.is_cuda:
                out = out.pin_memory()
        if out.is_cuda != L.is_cuda or not out.is_contiguous() or tuple(out.shape) != (F_, 2, H, W):
            raise DvcError("colorize_clip: `out` must be a contiguous [F,2,H,W] tensor on the same side as L")
        fl = first_last_lab.contiguous() if first_last_lab is not None else None
        rc = self.lib.dvc_colorize_clip(self.h, _ptr(L), F_, H, W, float(temperature), _ptr(fl), _ptr(out),
                                        _stream(self.device))
        self._check(rc, "dvc_colorize_clip")
        return out

    def colorize_video_rgb8(self, frames, size, temperature=1e-10, first_last_lab=None, wls=(500.0, 4.0), out=None,
                            return_last=False):
        """test.py:68-120 end to end: uint8 frames [F,Hs,Ws,3] -> sRGB uint8 [K,F,size[0],size[1],3], one image per cached
        exemplar and frame.  Per frame: CenterPad + CenterCrop to `size`, Lab, 1/2, the networks (colorize_clip's
        recurrence), ab x2 * 1.25, the WLS filter (wls = (lambda, sigma_color), or None to skip it) and Lab -> sRGB, all
        in one pipelined call whose device memory does not grow with F.

        frames: pinned CPU or CUDA (a pageable CPU tensor is pinned first); `out` lives where frames live.
        first_last_lab: None (zeros, test.py:80) or [K,3,size[0]/2,size[1]/2].  return_last=True also returns the
        recurrence state after the last frame, cat(L, ab) at half resolution [K,3,size[0]/2,size[1]/2] on the same side
        as frames: passed as the next call's first_last_lab it continues the clip exactly (chunked streaming)."""
        from dvc.prepost import centerpad_geometry

        if not (isinstance(frames, torch.Tensor) and frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[3] == 3):
            raise DvcError("colorize_video_rgb8: expected a uint8 tensor [F,Hs,Ws,3]")
        frames = frames.contiguous()
        if not frames.is_cuda and not frames.is_pinned():
            frames = frames.pin_memory()
        F_, Hs, Ws, _ = frames.shape
        Ho, Wo = int(size[0]), int(size[1])
        Hr, Wr, oy, ox = centerpad_geometry(Hs, Ws, (Ho, Wo))
        K = self.n_exemplars

        def host_or_device(shape, dtype):
            t = torch.empty(*shape, dtype=dtype, device=frames.device)
            return t if frames.is_cuda else t.pin_memory()

        if out is None:
            out = host_or_device((K, F_, Ho, Wo, 3), torch.uint8)
        if (out.is_cuda != frames.is_cuda or out.dtype != torch.uint8 or not out.is_contiguous()
                or tuple(out.shape) != (K, F_, Ho, Wo, 3)):
            raise DvcError("colorize_video_rgb8: `out` must be a contiguous uint8 [K,F,H,W,3] tensor on the same side as frames")
        fl = None
        if first_last_lab is not None:
            fl = first_last_lab.to(torch.float32).contiguous()
            if tuple(fl.shape) != (K, 3, Ho // 2, Wo // 2):
                raise DvcError("colorize_video_rgb8: first_last_lab must be [K,3,H/2,W/2]")
        last = host_or_device((K, 3, Ho // 2, Wo // 2), torch.float32) if return_last else None
        lam, sigma = (0.0, 1.0) if wls is None else (float(wls[0]), float(wls[1]))
        rc = self.lib.dvc_colorize_video_rgb8(self.h, _ptr(frames), F_, Hs, Ws, Hr, Wr, oy, ox, Ho, Wo, float(temperature), _ptr(fl),
                                              0 if wls is None else 1, lam, sigma, _ptr(out), _ptr(last), _stream(self.device))
        self._check(rc, "dvc_colorize_video_rgb8")
        return (out, last) if return_last else out

    # ---- several clips in one pass, clip s against exemplar slot s (set_exemplars with one image per clip) -----------
    def colorize_frames_clips(self, IA_l, last, temperature=1e-10, want_warp=False):
        """Frame s of IA_l [S,1,H,W] against cached exemplar slot s with last [S,3,H,W] -> ab [S,2,H,W]
        (, warp [S,3,H,W], sim [S,1,H,W]): colorize_frames once per clip, batched."""
        IA_l, last = _dev_f32(IA_l, "IA_l"), _dev_f32(last, "last")
        S, c1, H, W = IA_l.shape
        if c1 != 1 or tuple(last.shape) != (S, 3, H, W):
            raise DvcError("colorize_frames_clips: IA_l must be [S,1,H,W] and last [S,3,H,W]")
        ab = torch.empty(S, 2, H, W, device=IA_l.device, dtype=torch.float32)
        warp = torch.empty(S, 3, H, W, device=IA_l.device, dtype=torch.float32) if want_warp else None
        sim = torch.empty(S, 1, H, W, device=IA_l.device, dtype=torch.float32) if want_warp else None
        rc = self.lib.dvc_colorize_frames_clips(self.h, _ptr(IA_l), _ptr(last), S, H, W, float(temperature), _ptr(ab), _ptr(warp),
                                                _ptr(sim), _stream(IA_l.device))
        self._check(rc, "dvc_colorize_frames_clips")
        return (ab, warp, sim) if want_warp else ab

    def colorize_clips(self, L, temperature=1e-10, first_last_lab=None, out=None):
        """L [S,F,1,H,W] -> ab [S,F,2,H,W]: colorize_clip for S clips in one pass, clip s against exemplar slot s with its own
        recurrence.  first_last_lab: None (zeros) or [S,3,H,W].  L pinned on the host or on the device; `out` lives where
        L lives."""
        if L.dtype != torch.float32 or L.dim() != 5 or L.shape[2] != 1:
            raise DvcError("colorize_clips takes a float32 [S,F,1,H,W] tensor")
        L = L.contiguous()
        S, F_, _, H, W = L.shape
        if out is None:
            out = torch.empty(S, F_, 2, H, W, dtype=torch.float32, device=L.device)
            if not L.is_cuda:
                out = out.pin_memory()
        if out.is_cuda != L.is_cuda or not out.is_contiguous() or tuple(out.shape) != (S, F_, 2, H, W):
            raise DvcError("colorize_clips: `out` must be a contiguous [S,F,2,H,W] tensor on the same side as L")
        fl = None
        if first_last_lab is not None:
            fl = first_last_lab.to(torch.float32).contiguous()
            if tuple(fl.shape) != (S, 3, H, W):
                raise DvcError("colorize_clips: first_last_lab must be [S,3,H,W]")
        rc = self.lib.dvc_colorize_clips(self.h, _ptr(L), F_, H, W, float(temperature), _ptr(fl), S, _ptr(out), _stream(self.device))
        self._check(rc, "dvc_colorize_clips")
        return out

    def colorize_videos_rgb8(self, clips, size, temperature=1e-10, first_last_lab=None, wls=(500.0, 4.0), out=None,
                             return_last=False):
        """colorize_video_rgb8 for S clips in one pass: clips is a list of S uint8 tensors [F,Hs_s,Ws_s,3] (one F, source
        sizes may differ), clip s against exemplar slot s -> sRGB uint8 [S,F,size[0],size[1],3].  CenterPad's geometry is
        computed per clip.  The clips are all pinned CPU or all CUDA (pageable CPU tensors are pinned first); `out` lives
        where they live.  first_last_lab / the returned last state: [S,3,size[0]/2,size[1]/2], as in colorize_video_rgb8."""
        from dvc.prepost import centerpad_geometry

        clips = list(clips)
        if not clips or not all(isinstance(f, torch.Tensor) and f.dtype == torch.uint8 and f.dim() == 4 and f.shape[3] == 3
                                for f in clips):
            raise DvcError("colorize_videos_rgb8: expected a list of uint8 tensors [F,Hs,Ws,3]")
        on_device = clips[0].is_cuda
        if any(f.is_cuda != on_device for f in clips) or len({f.shape[0] for f in clips}) != 1:
            raise DvcError("colorize_videos_rgb8: the clips must have the same frame count and all live on the host or all on the device")
        clips = [f.contiguous() for f in clips]
        if not on_device:
            clips = [f if f.is_pinned() else f.pin_memory() for f in clips]
        S, F_ = len(clips), clips[0].shape[0]
        Ho, Wo = int(size[0]), int(size[1])
        geom = []
        for f in clips:
            Hs, Ws = f.shape[1], f.shape[2]
            geom += [Hs, Ws, *centerpad_geometry(Hs, Ws, (Ho, Wo))]

        def host_or_device(shape, dtype):
            t = torch.empty(*shape, dtype=dtype, device=clips[0].device)
            return t if on_device else t.pin_memory()

        if out is None:
            out = host_or_device((S, F_, Ho, Wo, 3), torch.uint8)
        if (out.is_cuda != on_device or out.dtype != torch.uint8 or not out.is_contiguous()
                or tuple(out.shape) != (S, F_, Ho, Wo, 3)):
            raise DvcError("colorize_videos_rgb8: `out` must be a contiguous uint8 [S,F,H,W,3] tensor on the same side as the clips")
        fl = None
        if first_last_lab is not None:
            fl = first_last_lab.to(torch.float32).contiguous()
            if tuple(fl.shape) != (S, 3, Ho // 2, Wo // 2):
                raise DvcError("colorize_videos_rgb8: first_last_lab must be [S,3,H/2,W/2]")
        last = host_or_device((S, 3, Ho // 2, Wo // 2), torch.float32) if return_last else None
        lam, sigma = (0.0, 1.0) if wls is None else (float(wls[0]), float(wls[1]))
        ptrs = (ctypes.c_void_p * S)(*[f.data_ptr() for f in clips])
        g = (ctypes.c_int * (6 * S))(*geom)
        rc = self.lib.dvc_colorize_videos_rgb8(self.h, S, ptrs, F_, g, Ho, Wo, float(temperature), _ptr(fl), 0 if wls is None else 1,
                                               lam, sigma, _ptr(out), _ptr(last), _stream(self.device))
        self._check(rc, "dvc_colorize_videos_rgb8")
        return (out, last) if return_last else out

    # ---- several clips in one pass, several exemplars each: K[s] rows per clip, R = sum(K) rows in all -------------------
    # Row r is one (clip, exemplar) pair, the rows of clip s are contiguous and row r runs against cached exemplar slot r
    # (set_exemplars with the R images in row order).  Every K[s] = 1 is the several-clip call, one clip the K-exemplar call.
    @staticmethod
    def _counts(K, S, what):
        K = [int(k) for k in K]
        if len(K) != S:
            raise DvcError(f"{what}: K must give one exemplar count per clip ({S} clips, {len(K)} counts)")
        return K, (ctypes.c_int * S)(*K)

    def colorize_frames_clips_exemplars(self, IA_l, K, last, temperature=1e-10, want_warp=False):
        """Frame s of IA_l [S,1,H,W] against the K[s] exemplar slots of clip s, last [R,3,H,W] -> ab [R,2,H,W]
        (, warp [R,3,H,W], sim [R,1,H,W])."""
        IA_l, last = _dev_f32(IA_l, "IA_l"), _dev_f32(last, "last")
        S, c1, H, W = IA_l.shape
        K, ck = self._counts(K, S, "colorize_frames_clips_exemplars")
        R = sum(K)
        if c1 != 1 or tuple(last.shape) != (R, 3, H, W):
            raise DvcError("colorize_frames_clips_exemplars: IA_l must be [S,1,H,W] and last [R,3,H,W], R = sum(K)")
        ab = torch.empty(R, 2, H, W, device=IA_l.device, dtype=torch.float32)
        warp = torch.empty(R, 3, H, W, device=IA_l.device, dtype=torch.float32) if want_warp else None
        sim = torch.empty(R, 1, H, W, device=IA_l.device, dtype=torch.float32) if want_warp else None
        rc = self.lib.dvc_colorize_frames_clips_exemplars(self.h, _ptr(IA_l), _ptr(last), S, ck, H, W, float(temperature), _ptr(ab),
                                                          _ptr(warp), _ptr(sim), _stream(IA_l.device))
        self._check(rc, "dvc_colorize_frames_clips_exemplars")
        return (ab, warp, sim) if want_warp else ab

    def colorize_clips_exemplars(self, L, K, temperature=1e-10, first_last_lab=None, out=None):
        """L [S,F,1,H,W] -> ab [R,F,2,H,W]: colorize_clips with K[s] exemplars for clip s, each row with its own recurrence.
        first_last_lab: None (zeros) or [R,3,H,W].  L pinned on the host or on the device; `out` lives where L lives."""
        if L.dtype != torch.float32 or L.dim() != 5 or L.shape[2] != 1:
            raise DvcError("colorize_clips_exemplars takes a float32 [S,F,1,H,W] tensor")
        L = L.contiguous()
        S, F_, _, H, W = L.shape
        K, ck = self._counts(K, S, "colorize_clips_exemplars")
        R = sum(K)
        if out is None:
            out = torch.empty(R, F_, 2, H, W, dtype=torch.float32, device=L.device)
            if not L.is_cuda:
                out = out.pin_memory()
        if out.is_cuda != L.is_cuda or not out.is_contiguous() or tuple(out.shape) != (R, F_, 2, H, W):
            raise DvcError("colorize_clips_exemplars: `out` must be a contiguous [R,F,2,H,W] tensor on the same side as L")
        fl = None
        if first_last_lab is not None:
            fl = first_last_lab.to(torch.float32).contiguous()
            if tuple(fl.shape) != (R, 3, H, W):
                raise DvcError("colorize_clips_exemplars: first_last_lab must be [R,3,H,W]")
        rc = self.lib.dvc_colorize_clips_exemplars(self.h, _ptr(L), F_, H, W, float(temperature), _ptr(fl), S, ck, _ptr(out),
                                                   _stream(self.device))
        self._check(rc, "dvc_colorize_clips_exemplars")
        return out

    def colorize_videos_exemplars_rgb8(self, clips, K, size, temperature=1e-10, first_last_lab=None, wls=(500.0, 4.0), out=None,
                                       return_last=False):
        """colorize_videos_rgb8 with K[s] exemplars for clip s: clips is a list of S uint8 tensors [F,Hs_s,Ws_s,3] -> sRGB
        uint8 [R,F,size[0],size[1],3], row r of clip s drawn with that clip's luminance and WLS guide.  first_last_lab / the
        returned last state: [R,3,size[0]/2,size[1]/2]; the rest as colorize_videos_rgb8."""
        from dvc.prepost import centerpad_geometry

        clips = list(clips)
        if not clips or not all(isinstance(f, torch.Tensor) and f.dtype == torch.uint8 and f.dim() == 4 and f.shape[3] == 3
                                for f in clips):
            raise DvcError("colorize_videos_exemplars_rgb8: expected a list of uint8 tensors [F,Hs,Ws,3]")
        on_device = clips[0].is_cuda
        if any(f.is_cuda != on_device for f in clips) or len({f.shape[0] for f in clips}) != 1:
            raise DvcError("colorize_videos_exemplars_rgb8: the clips must have the same frame count and all live on the host or all "
                           "on the device")
        clips = [f.contiguous() for f in clips]
        if not on_device:
            clips = [f if f.is_pinned() else f.pin_memory() for f in clips]
        S, F_ = len(clips), clips[0].shape[0]
        K, ck = self._counts(K, S, "colorize_videos_exemplars_rgb8")
        R = sum(K)
        Ho, Wo = int(size[0]), int(size[1])
        geom = []
        for f in clips:
            Hs, Ws = f.shape[1], f.shape[2]
            geom += [Hs, Ws, *centerpad_geometry(Hs, Ws, (Ho, Wo))]

        def host_or_device(shape, dtype):
            t = torch.empty(*shape, dtype=dtype, device=clips[0].device)
            return t if on_device else t.pin_memory()

        if out is None:
            out = host_or_device((R, F_, Ho, Wo, 3), torch.uint8)
        if (out.is_cuda != on_device or out.dtype != torch.uint8 or not out.is_contiguous()
                or tuple(out.shape) != (R, F_, Ho, Wo, 3)):
            raise DvcError("colorize_videos_exemplars_rgb8: `out` must be a contiguous uint8 [R,F,H,W,3] tensor on the same side as "
                           "the clips")
        fl = None
        if first_last_lab is not None:
            fl = first_last_lab.to(torch.float32).contiguous()
            if tuple(fl.shape) != (R, 3, Ho // 2, Wo // 2):
                raise DvcError("colorize_videos_exemplars_rgb8: first_last_lab must be [R,3,H/2,W/2]")
        last = host_or_device((R, 3, Ho // 2, Wo // 2), torch.float32) if return_last else None
        lam, sigma = (0.0, 1.0) if wls is None else (float(wls[0]), float(wls[1]))
        ptrs = (ctypes.c_void_p * S)(*[f.data_ptr() for f in clips])
        g = (ctypes.c_int * (6 * S))(*geom)
        rc = self.lib.dvc_colorize_videos_exemplars_rgb8(self.h, S, ck, ptrs, F_, g, Ho, Wo, float(temperature), _ptr(fl),
                                                         0 if wls is None else 1, lam, sigma, _ptr(out), _ptr(last), _stream(self.device))
        self._check(rc, "dvc_colorize_videos_exemplars_rgb8")
        return (out, last) if return_last else out

    # ---- output at the source resolution: the window's chroma on each source frame's own luminance -------------------------
    def ab_to_source(self, ab, geometry, size):
        """The window ab [...,Ho,Wo] (CUDA float32, size = (Ho, Wo)) resampled bilinearly onto the source footprint of
        geometry = (Hs, Ws, Hr, Wr, oy, ox): [...,h,w] (include/dvc.h: dvc_ab_to_source)."""
        ab = _dev_f32(ab, "ab_to_source input")
        Ho, Wo = int(size[0]), int(size[1])
        if ab.dim() < 2 or tuple(ab.shape[-2:]) != (Ho, Wo):
            raise DvcError("ab_to_source: the planes must be [...,Ho,Wo] with (Ho, Wo) = size")
        g = [int(v) for v in geometry]
        _, _, h, w = source_footprint(*g, Ho, Wo)
        out = torch.empty(*ab.shape[:-2], h, w, device=ab.device, dtype=torch.float32)
        planes = ab.numel() // (Ho * Wo)
        self._check(self.lib.dvc_ab_to_source(self.h, _ptr(ab), planes, Ho, Wo, *g, _ptr(out), _stream(ab.device)), "dvc_ab_to_source")
        return out

    def colorize_videos_source_rgb8(self, clips, K, size, temperature=1e-10, first_last_lab=None, wls=(500.0, 4.0), out=None,
                                    return_last=False):
        """colorize_videos_exemplars_rgb8 with every frame at its source resolution: a list of S uint8 tensors
        [K[s],F,h_s,w_s,3], (h_s, w_s) the footprint of clip s's window (source_footprint), drawn with the source frame's own
        luminance and the network's chroma.  The networks still run at `size`; first_last_lab and the returned last state are
        [R,3,size[0]/2,size[1]/2] as there.  `out`: None or a list of S such tensors on the side where the clips live."""
        from dvc.prepost import centerpad_geometry

        what = "colorize_videos_source_rgb8"
        clips = list(clips)
        if not clips or not all(isinstance(f, torch.Tensor) and f.dtype == torch.uint8 and f.dim() == 4 and f.shape[3] == 3
                                for f in clips):
            raise DvcError(f"{what}: expected a list of uint8 tensors [F,Hs,Ws,3]")
        on_device = clips[0].is_cuda
        if any(f.is_cuda != on_device for f in clips) or len({f.shape[0] for f in clips}) != 1:
            raise DvcError(f"{what}: the clips must have the same frame count and all live on the host or all on the device")
        clips = [f.contiguous() for f in clips]
        if not on_device:
            clips = [f if f.is_pinned() else f.pin_memory() for f in clips]
        S, F_ = len(clips), clips[0].shape[0]
        K, ck = self._counts(K, S, what)
        R = sum(K)
        Ho, Wo = int(size[0]), int(size[1])
        geom, shapes = [], []
        for f, k in zip(clips, K):
            g = [f.shape[1], f.shape[2], *centerpad_geometry(f.shape[1], f.shape[2], (Ho, Wo))]
            _, _, h, w = source_footprint(*g, Ho, Wo)
            geom += g
            shapes.append((k, F_, h, w, 3))

        def host_or_device(shape, dtype):
            t = torch.empty(*shape, dtype=dtype, device=clips[0].device)
            return t if on_device else t.pin_memory()

        if out is None:
            out = [host_or_device(shp, torch.uint8) for shp in shapes]
        out = list(out)
        if len(out) != S or any(o.is_cuda != on_device or o.dtype != torch.uint8 or not o.is_contiguous() or tuple(o.shape) != shp
                                for o, shp in zip(out, shapes)):
            raise DvcError(f"{what}: `out` must be a list of contiguous uint8 [K[s],F,h_s,w_s,3] tensors (the footprints) on the "
                           "same side as the clips")
        fl = None
        if first_last_lab is not None:
            fl = first_last_lab.to(torch.float32).contiguous()
            if tuple(fl.shape) != (R, 3, Ho // 2, Wo // 2):
                raise DvcError(f"{what}: first_last_lab must be [R,3,H/2,W/2]")
        last = host_or_device((R, 3, Ho // 2, Wo // 2), torch.float32) if return_last else None
        lam, sigma = (0.0, 1.0) if wls is None else (float(wls[0]), float(wls[1]))
        ptrs = (ctypes.c_void_p * S)(*[f.data_ptr() for f in clips])
        optrs = (ctypes.c_void_p * S)(*[o.data_ptr() for o in out])
        g = (ctypes.c_int * (6 * S))(*geom)
        rc = self.lib.dvc_colorize_videos_source_rgb8(self.h, S, ck, ptrs, F_, g, Ho, Wo, float(temperature), _ptr(fl),
                                                      0 if wls is None else 1, lam, sigma, optrs, _ptr(last), _stream(self.device))
        self._check(rc, f"dvc_{what}")
        return (out, last) if return_last else out

    # ---- JPEG output (test.py:120): files byte-identical to Pillow's, only the compressed bytes leave the device ----------------
    def encode_jpeg_into(self, rgb, out, sizes, quality=75):
        """Encode the CUDA uint8 images rgb [B,H,W,3] into out [B,stride] uint8 and sizes [B] int64, both CUDA or pinned CPU
        tensors (include/dvc.h: dvc_encode_jpeg).  Asynchronous on the current stream."""
        if not (isinstance(rgb, torch.Tensor) and rgb.is_cuda and rgb.dtype == torch.uint8 and rgb.dim() == 4 and rgb.shape[3] == 3):
            raise DvcError("encode_jpeg: expected a CUDA uint8 tensor [B,H,W,3]")
        rgb = rgb.contiguous()
        B, H, W, _ = rgb.shape
        if (out.dtype != torch.uint8 or out.dim() != 2 or out.shape[0] != B or out.stride(1) != 1 or sizes.dtype != torch.int64
                or tuple(sizes.shape) != (B,) or not sizes.is_contiguous()):
            raise DvcError("encode_jpeg: out must be uint8 [B,stride] (rows contiguous) and sizes int64 [B]")
        rc = self.lib.dvc_encode_jpeg(self.h, _ptr(rgb), B, H, W, int(quality), _ptr(out), out.stride(0), _ptr(sizes),
                                      _stream(self.device))
        self._check(rc, "dvc_encode_jpeg")

    def encode_jpeg(self, rgb, quality=75):
        """The JFIF files of the CUDA uint8 images rgb [B,H,W,3] (or one [H,W,3]) as a list of bytes, equal to
        PIL.Image.fromarray(x).save(f, "JPEG", quality=quality).  Synchronises the current stream."""
        if rgb.dim() == 3:
            rgb = rgb.unsqueeze(0)
        B, H, W = rgb.shape[0], rgb.shape[1], rgb.shape[2]
        out = torch.empty(B, jpeg_max_bytes(H, W), dtype=torch.uint8).pin_memory()
        sizes = torch.empty(B, dtype=torch.int64).pin_memory()
        self.encode_jpeg_into(rgb, out, sizes, quality)
        torch.cuda.current_stream(self.device).synchronize()
        return [out[b, :int(sizes[b])].numpy().tobytes() for b in range(B)]

    def colorize_videos_jpeg(self, clips, K, size, quality=75, source_resolution=False, temperature=1e-10, first_last_lab=None,
                             wls=(500.0, 4.0), out=None, sizes=None, return_last=False):
        """colorize_videos_exemplars_rgb8 (window output) or colorize_videos_source_rgb8 (source_resolution=True) with every frame
        encoded as encode_jpeg encodes it, on the device (include/dvc.h: dvc_colorize_videos_jpeg).  Returns (slots, sizes): slots a
        list of S uint8 tensors [K[s],F,stride], sizes int64 [R,F]; jpeg_files(slots, sizes) cuts the files out.  stride is
        jpeg_max_bytes of the largest output frame.  `out` / `sizes`: None or such tensors on the side where the clips live
        (pinned CPU or CUDA).  first_last_lab and the returned last state as in the rgb8 calls ([R,3,size[0]/2,size[1]/2])."""
        from dvc.prepost import centerpad_geometry

        what = "colorize_videos_jpeg"
        clips = list(clips)
        if not clips or not all(isinstance(f, torch.Tensor) and f.dtype == torch.uint8 and f.dim() == 4 and f.shape[3] == 3
                                for f in clips):
            raise DvcError(f"{what}: expected a list of uint8 tensors [F,Hs,Ws,3]")
        on_device = clips[0].is_cuda
        if any(f.is_cuda != on_device for f in clips) or len({f.shape[0] for f in clips}) != 1:
            raise DvcError(f"{what}: the clips must have the same frame count and all live on the host or all on the device")
        clips = [f.contiguous() for f in clips]
        if not on_device:
            clips = [f if f.is_pinned() else f.pin_memory() for f in clips]
        S, F_ = len(clips), clips[0].shape[0]
        K, ck = self._counts(K, S, what)
        R = sum(K)
        Ho, Wo = int(size[0]), int(size[1])
        geom, stride = [], jpeg_max_bytes(Ho, Wo)
        for f in clips:
            g = [f.shape[1], f.shape[2], *centerpad_geometry(f.shape[1], f.shape[2], (Ho, Wo))]
            geom += g
            if source_resolution:
                _, _, h, w = source_footprint(*g, Ho, Wo)
                stride = max(stride, jpeg_max_bytes(h, w))

        def host_or_device(shape, dtype):
            t = torch.empty(*shape, dtype=dtype, device=clips[0].device)
            return t if on_device else t.pin_memory()

        if out is None:
            out = [host_or_device((k, F_, stride), torch.uint8) for k in K]
        out = list(out)
        if len(out) != S or any(o.dtype != torch.uint8 or not o.is_contiguous() or o.dim() != 3 or tuple(o.shape[:2]) != (k, F_)
                                for o, k in zip(out, K)) or len({o.shape[2] for o in out}) != 1:
            raise DvcError(f"{what}: `out` must be a list of contiguous uint8 [K[s],F,stride] tensors with one stride")
        if sizes is None:
            sizes = host_or_device((R, F_), torch.int64)
        if sizes.dtype != torch.int64 or not sizes.is_contiguous() or tuple(sizes.shape) != (R, F_):
            raise DvcError(f"{what}: sizes must be a contiguous int64 [R,F] tensor")
        fl = None
        if first_last_lab is not None:
            fl = first_last_lab.to(torch.float32).contiguous()
            if tuple(fl.shape) != (R, 3, Ho // 2, Wo // 2):
                raise DvcError(f"{what}: first_last_lab must be [R,3,H/2,W/2]")
        last = host_or_device((R, 3, Ho // 2, Wo // 2), torch.float32) if return_last else None
        lam, sigma = (0.0, 1.0) if wls is None else (float(wls[0]), float(wls[1]))
        ptrs = (ctypes.c_void_p * S)(*[f.data_ptr() for f in clips])
        optrs = (ctypes.c_void_p * S)(*[o.data_ptr() for o in out])
        g = (ctypes.c_int * (6 * S))(*geom)
        rc = self.lib.dvc_colorize_videos_jpeg(self.h, S, ck, ptrs, F_, g, Ho, Wo, float(temperature), _ptr(fl), 0 if wls is None else 1,
                                               lam, sigma, 1 if source_resolution else 0, int(quality), optrs, out[0].shape[2],
                                               _ptr(sizes), _ptr(last), _stream(self.device))
        self._check(rc, f"dvc_{what}")
        return (out, sizes, last) if return_last else (out, sizes)

    # ---- greyscale sources: one byte per pixel in, the sRGB calls' bytes out ------------------------------------------------------
    def colorize_videos_gray8(self, clips, K, size, temperature=1e-10, first_last_lab=None, wls=(500.0, 4.0), source_resolution=False,
                              quality=None, out=None, sizes=None, return_last=False):
        """The video calls for grey clips (include/dvc.h: dvc_colorize_videos_gray8): clips is a list of S uint8 tensors [F,Hs,Ws]
        (or [F,Hs,Ws,1]).  Returns exactly what the matching call returns for the clips with each byte repeated into R, G and B:
        colorize_videos_exemplars_rgb8 (window output), colorize_videos_source_rgb8 (source_resolution=True) or, when quality is
        given, colorize_videos_jpeg.  `out` / `sizes` are those calls' output arguments."""
        from dvc.prepost import centerpad_geometry

        what = "colorize_videos_gray8"
        clips = list(clips)
        if not clips or not all(isinstance(f, torch.Tensor) and f.dtype == torch.uint8 and (f.dim() == 3 or (f.dim() == 4 and f.shape[3] == 1))
                                for f in clips):
            raise DvcError(f"{what}: expected a list of uint8 tensors [F,Hs,Ws] (or [F,Hs,Ws,1])")
        clips = [f[..., 0] if f.dim() == 4 else f for f in clips]
        on_device = clips[0].is_cuda
        if any(f.is_cuda != on_device for f in clips) or len({f.shape[0] for f in clips}) != 1:
            raise DvcError(f"{what}: the clips must have the same frame count and all live on the host or all on the device")
        clips = [f.contiguous() for f in clips]
        if not on_device:
            clips = [f if f.is_pinned() else f.pin_memory() for f in clips]
        S, F_ = len(clips), clips[0].shape[0]
        K, ck = self._counts(K, S, what)
        R = sum(K)
        Ho, Wo = int(size[0]), int(size[1])
        geom, frame_sizes = [], []
        for f in clips:
            g = [f.shape[1], f.shape[2], *centerpad_geometry(f.shape[1], f.shape[2], (Ho, Wo))]
            geom += g
            frame_sizes.append(tuple(source_footprint(*g, Ho, Wo)[2:]) if source_resolution else (Ho, Wo))

        def host_or_device(shape, dtype):
            t = torch.empty(*shape, dtype=dtype, device=clips[0].device)
            return t if on_device else t.pin_memory()

        if quality is not None:  # colorize_videos_jpeg's slots and sizes
            stride = max(jpeg_max_bytes(h, w) for h, w in frame_sizes + [(Ho, Wo)])
            if out is None:
                out = [host_or_device((k, F_, stride), torch.uint8) for k in K]
            out = list(out)
            if len(out) != S or any(o.dtype != torch.uint8 or not o.is_contiguous() or o.dim() != 3 or tuple(o.shape[:2]) != (k, F_)
                                    for o, k in zip(out, K)) or len({o.shape[2] for o in out}) != 1:
                raise DvcError(f"{what}: `out` must be a list of contiguous uint8 [K[s],F,stride] tensors with one stride")
            if sizes is None:
                sizes = host_or_device((R, F_), torch.int64)
            if sizes.dtype != torch.int64 or not sizes.is_contiguous() or tuple(sizes.shape) != (R, F_):
                raise DvcError(f"{what}: sizes must be a contiguous int64 [R,F] tensor")
            per_clip, stride = out, out[0].shape[2]
        elif source_resolution:  # colorize_videos_source_rgb8's list of footprint-size clips
            shapes = [(k, F_, h, w, 3) for k, (h, w) in zip(K, frame_sizes)]
            if out is None:
                out = [host_or_device(shp, torch.uint8) for shp in shapes]
            out = list(out)
            if len(out) != S or any(o.is_cuda != on_device or o.dtype != torch.uint8 or not o.is_contiguous() or tuple(o.shape) != shp
                                    for o, shp in zip(out, shapes)):
                raise DvcError(f"{what}: `out` must be a list of contiguous uint8 [K[s],F,h_s,w_s,3] tensors (the footprints) on the "
                               "same side as the clips")
            per_clip, stride = out, 0
        else:  # colorize_videos_exemplars_rgb8's [R,F,Ho,Wo,3], handed over clip by clip
            if out is None:
                out = host_or_device((R, F_, Ho, Wo, 3), torch.uint8)
            if (out.is_cuda != on_device or out.dtype != torch.uint8 or not out.is_contiguous()
                    or tuple(out.shape) != (R, F_, Ho, Wo, 3)):
                raise DvcError(f"{what}: `out` must be a contiguous uint8 [R,F,H,W,3] tensor on the same side as the clips")
            per_clip, stride = list(torch.split(out, K)), 0
        fl = None
        if first_last_lab is not None:
            fl = first_last_lab.to(torch.float32).contiguous()
            if tuple(fl.shape) != (R, 3, Ho // 2, Wo // 2):
                raise DvcError(f"{what}: first_last_lab must be [R,3,H/2,W/2]")
        last = host_or_device((R, 3, Ho // 2, Wo // 2), torch.float32) if return_last else None
        lam, sigma = (0.0, 1.0) if wls is None else (float(wls[0]), float(wls[1]))
        ptrs = (ctypes.c_void_p * S)(*[f.data_ptr() for f in clips])
        optrs = (ctypes.c_void_p * S)(*[o.data_ptr() for o in per_clip])
        g = (ctypes.c_int * (6 * S))(*geom)
        rc = self.lib.dvc_colorize_videos_gray8(self.h, S, ck, ptrs, F_, g, Ho, Wo, float(temperature), _ptr(fl), 0 if wls is None else 1,
                                                lam, sigma, 1 if source_resolution else 0, 0 if quality is None else int(quality), optrs,
                                                stride, _ptr(sizes if quality is not None else None), _ptr(last), _stream(self.device))
        self._check(rc, f"dvc_{what}")
        res = (out, sizes) if quality is not None else (out,)
        res += (last,) if return_last else ()
        return res if len(res) > 1 else res[0]

    # ---- planar YUV 4:2:0 (I420): cv2's BT.601 conversions on the device, and video calls that take and give I420 frames ---------
    def i420_to_rgb8(self, yuv):
        """cv2.cvtColor(COLOR_YUV2RGB_I420) of a CUDA uint8 [B,3H/2,W] tensor (H, W even): uint8 [B,H,W,3]
        (include/dvc.h: dvc_i420_to_rgb8)."""
        if not (isinstance(yuv, torch.Tensor) and yuv.is_cuda and yuv.dtype == torch.uint8 and yuv.dim() == 3 and yuv.shape[1] % 3 == 0):
            raise DvcError("i420_to_rgb8: expected a CUDA uint8 tensor [B,3H/2,W]")
        yuv = yuv.contiguous()
        B, H, W = yuv.shape[0], yuv.shape[1] * 2 // 3, yuv.shape[2]
        out = torch.empty(B, H, W, 3, device=yuv.device, dtype=torch.uint8)
        self._check(self.lib.dvc_i420_to_rgb8(self.h, _ptr(yuv), B, H, W, _ptr(out), _stream(yuv.device)), "dvc_i420_to_rgb8")
        return out

    def rgb8_to_i420(self, rgb):
        """cv2.cvtColor(COLOR_RGB2YUV_I420) of a CUDA uint8 [B,H,W,3] tensor (H, W even): uint8 [B,3H/2,W]
        (include/dvc.h: dvc_rgb8_to_i420)."""
        if not (isinstance(rgb, torch.Tensor) and rgb.is_cuda and rgb.dtype == torch.uint8 and rgb.dim() == 4 and rgb.shape[3] == 3):
            raise DvcError("rgb8_to_i420: expected a CUDA uint8 tensor [B,H,W,3]")
        rgb = rgb.contiguous()
        B, H, W, _ = rgb.shape
        out = torch.empty(B, H * 3 // 2, W, device=rgb.device, dtype=torch.uint8)
        self._check(self.lib.dvc_rgb8_to_i420(self.h, _ptr(rgb), B, H, W, _ptr(out), _stream(rgb.device)), "dvc_rgb8_to_i420")
        return out

    def colorize_videos_i420(self, clips, K, size, temperature=1e-10, first_last_lab=None, wls=(500.0, 4.0), source_resolution=False,
                             out_format="rgb", out=None, return_last=False):
        """The video calls for I420 clips (include/dvc.h: dvc_colorize_videos_i420): clips is a list of S uint8 tensors
        [F,3Hs/2,Ws] (Hs, Ws even).  Returns a list of S tensors, clip s's [K[s],F,h,w,3] sRGB frames (out_format="rgb") or
        [K[s],F,3h/2,w] I420 frames (out_format="i420"), (h, w) = size, or the clip's footprint (source_footprint) with
        source_resolution.  The sRGB frames are exactly those of colorize_videos_exemplars_rgb8 (its rows split by clip) or
        colorize_videos_source_rgb8 for the clips converted by i420_to_rgb8, the I420 frames rgb8_to_i420 of them.
        first_last_lab and the returned last state are [R,3,size[0]/2,size[1]/2] as there.  `out`: None or such a list on the
        side where the clips live (pinned host or device)."""
        from dvc.prepost import centerpad_geometry

        what = "colorize_videos_i420"
        if out_format not in ("rgb", "i420"):
            raise DvcError(f'{what}: out_format must be "rgb" or "i420"')
        clips = list(clips)
        if not clips or not all(isinstance(f, torch.Tensor) and f.dtype == torch.uint8 and f.dim() == 3 and f.shape[1] % 3 == 0
                                for f in clips):
            raise DvcError(f"{what}: expected a list of uint8 tensors [F,3Hs/2,Ws]")
        on_device = clips[0].is_cuda
        if any(f.is_cuda != on_device for f in clips) or len({f.shape[0] for f in clips}) != 1:
            raise DvcError(f"{what}: the clips must have the same frame count and all live on the host or all on the device")
        clips = [f.contiguous() for f in clips]
        if not on_device:
            clips = [f if f.is_pinned() else f.pin_memory() for f in clips]
        S, F_ = len(clips), clips[0].shape[0]
        K, ck = self._counts(K, S, what)
        R = sum(K)
        Ho, Wo = int(size[0]), int(size[1])
        geom, shapes = [], []
        for f, k in zip(clips, K):
            Hs, Ws = f.shape[1] * 2 // 3, f.shape[2]
            g = [Hs, Ws, *centerpad_geometry(Hs, Ws, (Ho, Wo))]
            h, w = tuple(source_footprint(*g, Ho, Wo)[2:]) if source_resolution else (Ho, Wo)
            geom += g
            shapes.append((k, F_, h, w, 3) if out_format == "rgb" else (k, F_, h * 3 // 2, w))

        def host_or_device(shape, dtype):
            t = torch.empty(*shape, dtype=dtype, device=clips[0].device)
            return t if on_device else t.pin_memory()

        if out is None:
            out = [host_or_device(shp, torch.uint8) for shp in shapes]
        out = list(out)
        if len(out) != S or any(o.is_cuda != on_device or o.dtype != torch.uint8 or not o.is_contiguous() or tuple(o.shape) != shp
                                for o, shp in zip(out, shapes)):
            layout = "[K[s],F,h_s,w_s,3]" if out_format == "rgb" else "[K[s],F,3h_s/2,w_s]"
            raise DvcError(f"{what}: `out` must be a list of contiguous uint8 {layout} tensors on the same side as the clips")
        fl = None
        if first_last_lab is not None:
            fl = first_last_lab.to(torch.float32).contiguous()
            if tuple(fl.shape) != (R, 3, Ho // 2, Wo // 2):
                raise DvcError(f"{what}: first_last_lab must be [R,3,H/2,W/2]")
        last = host_or_device((R, 3, Ho // 2, Wo // 2), torch.float32) if return_last else None
        lam, sigma = (0.0, 1.0) if wls is None else (float(wls[0]), float(wls[1]))
        ptrs = (ctypes.c_void_p * S)(*[f.data_ptr() for f in clips])
        optrs = (ctypes.c_void_p * S)(*[o.data_ptr() for o in out])
        g = (ctypes.c_int * (6 * S))(*geom)
        rc = self.lib.dvc_colorize_videos_i420(self.h, S, ck, ptrs, F_, g, Ho, Wo, float(temperature), _ptr(fl), 0 if wls is None else 1,
                                               lam, sigma, 1 if source_resolution else 0, 1 if out_format == "i420" else 0, optrs,
                                               _ptr(last), _stream(self.device))
        self._check(rc, f"dvc_{what}")
        return (out, last) if return_last else out

    # ---- pre / post-processing around the nets (test.py:58,71,100-102) ----------------------------------
    def resize_half(self, x):
        """F.interpolate(x, scale_factor=0.5, mode="bilinear") for a CUDA [B,C,H,W] tensor with even H, W."""
        x = _dev_f32(x, "resize_half input")
        if x.data_ptr() % 8:  # a view at an odd float offset: dvc_resize_half loads pairs of floats and refuses it
            x = x.clone()
        B, C, H, W = x.shape
        out = torch.empty(B, C, H // 2, W // 2, device=x.device, dtype=torch.float32)
        self._check(self.lib.dvc_resize_half(self.h, _ptr(x), B * C, H, W, _ptr(out), _stream(x.device)), "dvc_resize_half")
        return out

    def upsample2_scaled(self, x, scale=1.25):
        """F.interpolate(x, scale_factor=2, mode="bilinear") * scale for a CUDA [B,C,h,w] tensor."""
        x = _dev_f32(x, "upsample2 input")
        B, C, h, w = x.shape
        out = torch.empty(B, C, 2 * h, 2 * w, device=x.device, dtype=torch.float32)
        self._check(self.lib.dvc_upsample2_scaled(self.h, _ptr(x), B * C, h, w, float(scale), _ptr(out), _stream(x.device)),
                    "dvc_upsample2_scaled")
        return out

    def lab_to_rgb8(self, l, ab):
        """batch_lab2rgb_transpose_mc (utils/util.py:140-151) for CUDA l [B,1,H,W] (centred) and ab [B,2,H,W]:
        uint8 [B,H,W,3] sRGB, computed in float64 like skimage.color.lab2rgb."""
        l, ab = _dev_f32(l, "lab_to_rgb8 l"), _dev_f32(ab, "lab_to_rgb8 ab")
        B, _, H, W = l.shape
        if tuple(ab.shape) != (B, 2, H, W) or l.shape[1] != 1:
            raise DvcError("lab_to_rgb8: expected l [B,1,H,W] and ab [B,2,H,W]")
        out = torch.empty(B, H, W, 3, device=l.device, dtype=torch.uint8)
        self._check(self.lib.dvc_lab_to_rgb8(self.h, _ptr(l), _ptr(ab), B, H, W, ctypes.c_void_p(out.data_ptr()), _stream(l.device)),
                    "dvc_lab_to_rgb8")
        return out

    def rgb8_to_lab(self, rgb):
        """RGB2Lab + ToTensor + Normalize of test.py:44-45 for a CUDA uint8 [B,H,W,3] tensor: float32 [B,3,H,W] with
        centred L, computed in float64 like skimage.color.rgb2lab."""
        if not (isinstance(rgb, torch.Tensor) and rgb.is_cuda and rgb.dtype == torch.uint8 and rgb.dim() == 4 and rgb.shape[3] == 3):
            raise DvcError("rgb8_to_lab: expected a CUDA uint8 tensor [B,H,W,3]")
        rgb = rgb.contiguous()
        B, H, W, _ = rgb.shape
        out = torch.empty(B, 3, H, W, device=rgb.device, dtype=torch.float32)
        self._check(self.lib.dvc_rgb8_to_lab(self.h, ctypes.c_void_p(rgb.data_ptr()), B, H, W, _ptr(out), _stream(rgb.device)),
                    "dvc_rgb8_to_lab")
        return out

    def contextual_loss_forward(self, X_features, Y_features, h=0.1, feature_centering=True):
        """ContextualLoss_forward.forward (models/ContextualLoss.py:82-126), value only: CUDA float32 [B,C,h,w] (or [B,C,N])
        feature maps -> loss [B]."""
        X, Y = _dev_f32(X_features, "contextual_loss X"), _dev_f32(Y_features, "contextual_loss Y")
        B, C = X.shape[0], X.shape[1]
        if Y.shape[0] != B or Y.shape[1] != C:
            raise DvcError("contextual_loss: X and Y must share batch size and feature depth")
        NX, NY = X[0, 0].numel(), Y[0, 0].numel()
        out = torch.empty(B, device=X.device, dtype=torch.float32)
        self._check(self.lib.dvc_contextual_loss_forward(self.h, _ptr(X), _ptr(Y), B, C, NX, NY, float(h), 1 if feature_centering else 0,
                                                         _ptr(out), _stream(X.device)), "dvc_contextual_loss_forward")
        return out

    def fgs_filter(self, guide, src, lam=500.0, sigma_color=4.0, lambda_attenuation=0.25, num_iter=3):
        """cv2.ximgproc.createFastGlobalSmootherFilter(guide, lam, sigma_color).filter(plane) for every plane of the
        CUDA float32 tensor src [P,H,W] with the CUDA uint8 guide [H,W] (test.py:105-112; defaults of test.py:32-33)."""
        src = _dev_f32(src, "fgs_filter src")
        if not (isinstance(guide, torch.Tensor) and guide.is_cuda and guide.dtype == torch.uint8 and guide.dim() == 2):
            raise DvcError("fgs_filter: the guide must be a CUDA uint8 [H,W] tensor")
        P, H, W = src.shape
        if tuple(guide.shape) != (H, W):
            raise DvcError("fgs_filter: guide and planes differ in size")
        guide = guide.contiguous()
        out = torch.empty_like(src)
        self._check(self.lib.dvc_fgs_filter(self.h, ctypes.c_void_p(guide.data_ptr()), _ptr(src), P, H, W, float(lam), float(sigma_color),
                                            float(lambda_attenuation), int(num_iter), _ptr(out), _stream(src.device)), "dvc_fgs_filter")
        return out

    def l_to_guide8(self, l):
        """uint8(uncenter_l(L) * 255 / 100) (test.py:106) for a CUDA float32 [H,W] centred-luminance plane."""
        l = _dev_f32(l, "l_to_guide8 input")
        H, W = l.shape[-2:]
        out = torch.empty(H, W, device=l.device, dtype=torch.uint8)
        self._check(self.lib.dvc_l_to_guide8(self.h, _ptr(l), H, W, ctypes.c_void_p(out.data_ptr()), _stream(l.device)), "dvc_l_to_guide8")
        return out

    def centerpad_rgb8(self, rgb, size):
        """CenterPad(size) + CenterCrop(size) of test.py:44-46 for a CUDA uint8 [H,W,3] image -> uint8 [size[0],size[1],3]."""
        from dvc.prepost import centerpad_geometry

        if not (isinstance(rgb, torch.Tensor) and rgb.is_cuda and rgb.dtype == torch.uint8 and rgb.dim() == 3 and rgb.shape[2] == 3):
            raise DvcError("centerpad_rgb8: expected a CUDA uint8 tensor [H,W,3]")
        rgb = rgb.contiguous()
        Hs, Ws, _ = rgb.shape
        Hr, Wr, oy, ox = centerpad_geometry(Hs, Ws, size)
        out = torch.empty(size[0], size[1], 3, device=rgb.device, dtype=torch.uint8)
        self._check(self.lib.dvc_resize_antialias_crop_rgb8(self.h, ctypes.c_void_p(rgb.data_ptr()), Hs, Ws, Hr, Wr, oy, ox,
                                                            ctypes.c_void_p(out.data_ptr()), size[0], size[1], _stream(rgb.device)),
                    "dvc_resize_antialias_crop_rgb8")
        return out

    # ---- query-row-sharded correlation: peer-mapped result buffers (CUDA IPC) ----------------------------
    def peer_buffer_create(self, nbytes):
        """(device pointer, 64-byte IPC handle) of a fresh zeroed cudaMalloc allocation other ranks can map."""
        ptr, handle = ctypes.c_void_p(0), ctypes.create_string_buffer(64)
        self._check(self.lib.dvc_peer_buffer_create(self.h, int(nbytes), ctypes.byref(ptr), handle), "dvc_peer_buffer_create")
        return ptr.value, handle.raw

    def peer_buffer_open(self, handle):
        ptr = ctypes.c_void_p(0)
        self._check(self.lib.dvc_peer_buffer_open(self.h, ctypes.create_string_buffer(bytes(handle), 64), ctypes.byref(ptr)),
                    "dvc_peer_buffer_open")
        return ptr.value

    def peer_buffer_close(self, ptr):
        self._check(self.lib.dvc_peer_buffer_close(self.h, ctypes.c_void_p(ptr)), "dvc_peer_buffer_close")

    def peer_buffer_destroy(self, ptr):
        self._check(self.lib.dvc_peer_buffer_destroy(self.h, ctypes.c_void_p(ptr)), "dvc_peer_buffer_destroy")

    def corr_set_peer_outputs(self, y4_ptrs=(), sim_ptrs=(), row0=0):
        """Route the result rows of the next corr_softmax_warp calls into these peer buffers as well (empty = off)."""
        n = len(y4_ptrs)
        ya = (ctypes.c_void_p * max(n, 1))(*[ctypes.c_void_p(p) for p in y4_ptrs])
        sa = (ctypes.c_void_p * max(n, 1))(*[ctypes.c_void_p(p) for p in sim_ptrs])
        self._check(self.lib.dvc_corr_set_peer_outputs(self.h, n, ya, sa, int(row0)), "dvc_corr_set_peer_outputs")

    def raw_view(self, ptr, numel):
        """float32 tensor view of `numel` elements at a device pointer owned by the library."""
        return _raw_view(ptr, numel, self.device)

    # ---- multi-GPU: exemplar operands as one flat buffer (broadcast with torch.distributed / NCCL) ----
    def exemplar_pack_size(self, H, W):
        return int(self.lib.dvc_exemplar_pack_size(self.h, H, W))

    def exemplar_export(self, H, W):
        buf = torch.empty(self.exemplar_pack_size(H, W), device=self.device, dtype=torch.float32)
        self._check(self.lib.dvc_exemplar_export(self.h, _ptr(buf), buf.numel(), _stream(self.device)),
                    "dvc_exemplar_export")
        return buf

    def exemplar_import(self, buf, H, W):
        buf = _dev_f32(buf, "exemplar pack")
        self._check(self.lib.dvc_exemplar_import(self.h, _ptr(buf), buf.numel(), H, W, _stream(self.device)),
                    "dvc_exemplar_import")
        self.n_exemplars = 1

    # ---- debug hooks ---------------------------------------------------------------------------------
    def debug_flag(self, name, value):
        self._check(self.lib.dvc_debug_set_flag(self.h, name.encode(), int(value)), "dvc_debug_set_flag")

    def debug_conv2d(self, net, name, x, cout, dil=1, stride=1, act=0, slope=0.0, reflect=False, upconv=False,
                     fuse_tail=False, in_bound=None, out_planes=False, add=None, want_stats=False):
        """One convolution layer (weights `name` of `net`) on a CUDA NCHW tensor through the engine the layer programs
        use (include/dvc.h: dvc_debug_conv2d).  Returns y or (y, stats [B,cout,2] float64).

        in_bound: a bound of max |x| (default: x.abs().max()), or a negative value for the first layers (Cin <= 8), whose
        max |x| is then measured on the device; out_planes=True on a first layer needs that measured bound."""
        x = _dev_f32(x, "debug_conv2d input")
        B, _, H, W = x.shape
        Ho, Wo = (2 * H, 2 * W) if upconv else ((H + stride - 1) // stride, (W + stride - 1) // stride)
        y = torch.empty(B, 2 if fuse_tail else cout, Ho, Wo, device=x.device, dtype=torch.float32)
        st = torch.zeros(B, cout, 2, device=x.device, dtype=torch.float64) if want_stats else None
        bound = float(x.abs().max()) if in_bound is None else float(in_bound)
        add = _dev_f32(add, "debug_conv2d addend") if add is not None else None
        rc = self.lib.dvc_debug_conv2d(self.h, net, name.encode(), _ptr(x), B, H, W, dil, stride, act, float(slope),
                                       1 if reflect else 0, 1 if upconv else 0, 1 if fuse_tail else 0, bound,
                                       1 if out_planes else 0, _ptr(add), _ptr(y), _ptr(st), _stream(x.device))
        self._check(rc, "dvc_debug_conv2d")
        return (y, st) if want_stats else y

    def debug_buffer(self, name, act=True, keep_border=False, fp16=False):
        """Copy of an internal workspace.  act=True: padded NHWC activation -> interior as NCHW [B,C,H,W].

        keep_border=True returns the padded tensor [B,C,H+2P,W+2P].  An activation stored as fp16 hi/lo planes of
        value * 2^e comes back as hi + lo in those scaled units (the exponent lives in the layer program); fp16=True
        asks for those planes also when the buffer keeps an fp32 plane beside them."""
        ptr, nbytes, sig = ctypes.c_void_p(0), ctypes.c_int64(0), (ctypes.c_int * 5)()
        self._check(self.lib.dvc_debug_get_buffer(self.h, name.encode(), ctypes.byref(ptr), ctypes.byref(nbytes), sig),
                    "dvc_debug_get_buffer")
        torch.cuda.synchronize(self.device)
        flat = _raw_view(ptr.value, nbytes.value // 4, self.device).clone()
        if not act:
            return flat
        B, H, W, C, P = list(sig)
        split = P < 0  # hi/lo planes of a tensor-core activation are stored back to back
        if split:
            P = -1 - P
        mode16, P = divmod(P, 1000)  # 2: fp16 hi/lo planes of value * 2^e only; 3: an fp32 plane followed by them
        n = B * (H + 2 * P) * (W + 2 * P) * C
        if fp16 and mode16 not in (2, 3):
            raise DvcError(f"debug_buffer({name}): no fp16 planes in this buffer")
        if mode16 == 2 or (mode16 == 3 and fp16):
            halves = flat.view(torch.float16)[(2 * n if mode16 == 3 else 0):]
            t = halves[:n].float() + halves[n:2 * n].float()
        else:
            t = flat[:n] + flat[n:2 * n] if split else flat[:n]
        t = t.view(B, H + 2 * P, W + 2 * P, C)
        if not keep_border:
            t = t[:, P:P + H, P:P + W, :]
        return t.permute(0, 3, 1, 2).contiguous()

    # ---- introspection ---------------------------------------------------------------------------
    def launch_count(self, reset=False):
        return int(self.lib.dvc_launch_count(self.h, 1 if reset else 0))

    def profile_corr(self, enable=True):
        self._check(self.lib.dvc_profile_corr(self.h, 1 if enable else 0), "dvc_profile_corr")

    def profile_conv(self, enable=True):
        self._check(self.lib.dvc_profile_conv(self.h, 1 if enable else 0), "dvc_profile_conv")

    def conv_profile(self, variant=0, reset=False):
        """(launches, total ms, total algorithmic FLOPs) of the recorded tensor-core conv launches of `variant`."""
        ms, fl = ctypes.c_double(0), ctypes.c_double(0)
        n = self.lib.dvc_conv_profile(self.h, variant, 1 if reset else 0, ctypes.byref(ms), ctypes.byref(fl))
        return int(n), ms.value, fl.value

    def corr_mean_ms(self, reset=True):
        return float(self.lib.dvc_corr_mean_ms(self.h, 1 if reset else 0))


def _raw_view(ptr, n_floats, device):
    """float32 tensor aliasing raw device memory (debug only) via the CUDA array interface."""

    class _Holder:
        pass

    h = _Holder()
    h.__cuda_array_interface__ = {"shape": (n_floats,), "typestr": "<f4", "data": (ptr, False), "version": 2}
    return torch.as_tensor(h, device=device)


def source_footprint(Hs, Ws, Hr, Wr, oy, ox, Ho, Wo):
    """(y0, x0, h, w): the source pixels of geometry (Hs, Ws, Hr, Wr, oy, ox) whose centres fall inside the (Ho, Wo) window's
    extent, the size of colorize_videos_source_rgb8's output frames (include/dvc.h: dvc_source_footprint).  Needs no GPU."""
    fp = (ctypes.c_int * 4)()
    rc = load_library().dvc_source_footprint(int(Hs), int(Ws), int(Hr), int(Wr), int(oy), int(ox), int(Ho), int(Wo), fp)
    if rc != 0:
        raise DvcError(f"dvc_source_footprint failed ({rc}): geometry {(Hs, Ws, Hr, Wr, oy, ox)} has no source pixel inside the "
                       f"{Ho}x{Wo} window, or a size < 1")
    return tuple(fp)


def resize_taps(in_len, out_len):
    """The Gaussian taps CenterPad's anti-aliasing filter gives an axis resized from in_len to out_len pixels, as the host code
    hands them to the kernel (dvc_debug_resize_taps; needs no GPU): a list of 2 * radius + 1 floats, empty without a filter."""
    lib = load_library()
    radius = ctypes.c_int(0)
    rc = lib.dvc_debug_resize_taps(int(in_len), int(out_len), None, 0, ctypes.byref(radius))  # -2: radius set, taps do not fit
    buf = (ctypes.c_double * (2 * radius.value + 1 if rc == -2 else 0))()
    if rc == -2:
        rc = lib.dvc_debug_resize_taps(int(in_len), int(out_len), buf, len(buf), ctypes.byref(radius))
    if rc != 0:
        raise DvcError(f"dvc_debug_resize_taps({in_len}, {out_len}) failed ({rc})")
    return list(buf)


def jpeg_max_bytes(h, w):
    """Upper bound on the size of an h x w JPEG file of encode_jpeg for any content and quality (include/dvc.h:
    dvc_jpeg_max_bytes).  Needs no GPU."""
    n = int(load_library().dvc_jpeg_max_bytes(int(h), int(w)))
    if n < 0:
        raise DvcError(f"dvc_jpeg_max_bytes failed ({n}): {h}x{w} is outside the encoder's sizes")
    return n


def jpeg_files(slots, sizes):
    """The files of colorize_videos_jpeg: slots (S tensors [K[s],F,stride]) and sizes [R,F] -> [R][F] lists of bytes, row-major
    over the clips' rows."""
    sizes = sizes.cpu()
    files = []
    for o in slots:
        o = o.cpu()
        for r in range(o.shape[0]):
            files.append([o[r, t, :int(sizes[len(files), t])].numpy().tobytes() for t in range(o.shape[1])])
    return files


_contexts = {}


def get_context(device=None):
    """Process-wide context of a device (shared by the three drop-in modules, like test.py:147-166)."""
    if device is None:
        device = torch.cuda.current_device() if torch.cuda.is_available() else 0
    idx = device if isinstance(device, int) else (torch.device(device).index or 0)
    if idx not in _contexts:
        _contexts[idx] = Context(idx)
    return _contexts[idx]
