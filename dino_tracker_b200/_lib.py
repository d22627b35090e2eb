"""ctypes binding of libdinotrk.so (include/dinotrk.h).  There is NO fallback: if the CUDA library is
missing or fails to load, importing the product path raises."""
import ctypes
import os
import struct
import warnings
from ctypes import POINTER, Structure, c_char_p, c_float, c_int, c_size_t, c_ulonglong, c_void_p

import torch

from . import build as _build

_LIB = None


class Geom(Structure):
    _fields_ = [("H", c_int), ("W", c_int), ("patch", c_int), ("stride", c_int), ("radius", c_int),
                ("h", c_int), ("w", c_int)]


class HeadWeights(Structure):
    _fields_ = [("w1", c_float * 9 * 16), ("b1", c_float * 16), ("w2", c_float * 9 * 16), ("b2", c_float)]


class Features(Structure):
    _fields_ = [("tpc", c_void_p), ("norms", c_void_p), ("hi", c_void_p), ("lo", c_void_p), ("T", c_int), ("C", c_int),
                ("q8", c_void_p), ("q_fac", c_void_p), ("q_rho", c_void_p)]


class VitConfig(Structure):
    _fields_ = [("depth", c_int), ("dim", c_int), ("heads", c_int), ("tap_layer", c_int), ("patch", c_int), ("stride", c_int),
                ("attn_materialized", c_int), ("gemm_f16", c_int), ("gemm_pair", c_int)]


class VitWeights(Structure):
    _fields_ = [("patch_w", c_void_p), ("patch_b", c_void_p), ("cls_pos", c_void_p), ("pos", c_void_p),
                ("blocks", POINTER(c_void_p))]


class FlowVideo(Structure):
    _fields_ = [("fwd", c_void_p), ("bwd", c_void_p), ("T", c_int), ("H", c_int), ("W", c_int)]


RAFT_NCONV = 45   # include/dinotrk.h DINOTRK_RAFT_NCONV


class RaftWeights(Structure):
    _fields_ = [("w_hi", c_void_p * RAFT_NCONV), ("w_lo", c_void_p * RAFT_NCONV), ("bias", c_void_p * RAFT_NCONV),
                ("scale", c_float * RAFT_NCONV)]


class DinotrkError(RuntimeError):
    pass


# every exported symbol of include/dinotrk.h: name -> (restype, argtypes)
_P = c_void_p
SIGNATURES = {
    "dinotrk_version": (c_int, []),
    "dinotrk_last_error": (c_char_p, []),
    "dinotrk_launch_count": (c_ulonglong, []),
    "dinotrk_make_geom": (c_int, [c_int, c_int, c_int, c_int, c_int, POINTER(Geom)]),
    "dinotrk_pack_features": (c_int, [_P, _P, _P, c_int, c_int, c_int, _P]),
    "dinotrk_unpack_features": (c_int, [_P, _P, c_int, c_int, c_int, _P]),
    "dinotrk_token_norms": (c_int, [_P, _P, c_int, c_int, c_int, _P]),
    "dinotrk_sample_descriptors": (c_int, [_P, c_int, c_int, POINTER(Geom), _P, c_int, _P, c_int, c_int, _P, _P, _P]),
    "dinotrk_split_fp16": (c_int, [_P, _P, _P, c_size_t, _P]),
    "dinotrk_quantise_s8": (c_int, [_P, _P, c_size_t, c_int, c_int, _P, _P, _P, _P, _P]),
    "dinotrk_split_range": (c_int, [_P, c_size_t, _P, c_size_t, _P, _P]),
    "dinotrk_split_faithful": (c_int, [c_float, c_float, c_int]),
    "dinotrk_corr_track_workspace_bytes": (c_size_t, [c_int, c_int, c_int, POINTER(Geom)]),
    "dinotrk_corr_track": (c_int, [POINTER(Features), POINTER(Geom), POINTER(HeadWeights), _P, _P, _P, _P, _P, _P,
                                   c_int, c_int, c_int, _P, _P, c_int, c_int, _P, c_size_t, _P]),
    "dinotrk_corr_maps_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "dinotrk_map_stride": (c_int, [POINTER(Geom)]),
    "dinotrk_corr_maps": (c_int, [POINTER(Features), POINTER(Geom), _P, _P, _P, _P, _P, _P, c_int, c_int, c_int,
                                  _P, _P, c_size_t, _P]),
    "dinotrk_head": (c_int, [_P, c_int, POINTER(Geom), POINTER(HeadWeights), _P, _P, c_int, c_int, _P, _P, _P]),
    "dinotrk_sample_backward": (c_int, [c_int, c_int, POINTER(Geom), _P, c_int, _P, c_int, c_int, _P, _P, _P]),
    "dinotrk_track_backward_workspace_bytes": (c_size_t, [c_int, c_int, POINTER(Geom)]),
    "dinotrk_track_backward": (c_int, [POINTER(Features), POINTER(Geom), POINTER(HeadWeights), _P, _P, c_int, _P, _P, _P, _P, _P,
                                       _P, c_int, _P, _P, _P, c_size_t, _P]),
    "dinotrk_infer_workspace_bytes": (c_size_t, [c_int, c_int, POINTER(Geom), c_int, c_int]),
    "dinotrk_infer_set_overlap": (c_int, [c_int]),
    "dinotrk_infer_set_path": (c_int, [c_int]),
    "dinotrk_infer_set_coarse": (c_int, [c_int]),
    "dinotrk_infer_last_stats": (c_int, [POINTER(ctypes.c_longlong), c_int]),
    "dinotrk_infer_max_chunks": (c_size_t, [c_int, c_int, c_int]),
    "dinotrk_xw_coarse_keys_workspace_bytes": (c_size_t, [c_int, c_int, POINTER(Geom)]),
    "dinotrk_xw_coarse_keys": (c_int, [POINTER(Features), POINTER(Geom), _P, c_int, _P, _P, _P, _P, c_int, _P, _P, _P, c_size_t,
                                       _P]),
    "dinotrk_xw_coarse_keys_i8": (c_int, [POINTER(Features), POINTER(Geom), _P, _P, _P, c_int, _P, _P, _P, c_int, _P, _P, _P, _P,
                                          c_size_t, _P]),
    "dinotrk_xw_box_gemm": (c_int, [POINTER(Features), POINTER(Geom), _P, _P, c_int, _P, _P, _P, _P, c_int, c_int, _P, _P]),
    "dinotrk_infer_plan": (c_int, [c_int, c_int, c_int, _P, c_int, _P, _P, c_int, _P]),
    "dinotrk_infer_anchor_gcap": (c_int, [c_int, c_int]),
    "dinotrk_infer_plan_anchors": (c_int, [c_int, c_int, _P, _P, _P, c_int, c_int, _P, _P, c_int, _P]),
    "dinotrk_infer": (c_int, [POINTER(Features), POINTER(Geom), POINTER(HeadWeights), _P, c_int, c_float, c_float,
                              c_int, c_int, c_int, c_int, _P, _P, _P, _P, _P, c_size_t, _P]),
    "dinotrk_traj_cos_sims": (c_int, [_P, c_int, c_int, POINTER(Geom), _P, _P, c_int, _P, _P, c_size_t, _P]),
    "dinotrk_delta_workspace_bytes": (c_size_t, [c_int, c_int, c_int, POINTER(c_int)]),
    "dinotrk_delta_refine": (c_int, [_P, c_int, c_int, c_int, POINTER(c_int), POINTER(c_void_p), POINTER(c_void_p), _P,
                                     _P, _P, c_int, c_int, _P, _P, _P, c_size_t, _P]),
    "dinotrk_vit_workspace_bytes": (c_size_t, [POINTER(VitConfig), POINTER(Geom), c_int]),
    "dinotrk_vit_attention": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, _P, _P]),
    "dinotrk_vit_attention_f16": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, _P, _P]),
    "dinotrk_vit_stage": (c_int, [c_int, POINTER(VitConfig), POINTER(Geom), c_int, _P, _P, _P, _P, _P, _P, _P, _P, c_size_t,
                                  _P]),
    "dinotrk_vit_forward": (c_int, [_P, c_int, POINTER(Geom), POINTER(VitConfig), POINTER(VitWeights), _P, _P, c_size_t, _P]),
    "dinotrk_best_buddies_workspace_bytes": (c_size_t, [c_int, c_int]),
    "dinotrk_best_buddies_pairs": (c_int, [POINTER(Features), POINTER(Geom), _P, _P, c_int, _P, _P, _P, c_size_t, _P]),
    "dinotrk_bb_mutual": (c_int, [_P, _P, c_int, c_int, _P, _P]),
    "dinotrk_bb_nms": (c_int, [_P, c_int, POINTER(Geom), c_float, c_float, c_int, _P, _P, _P]),
    "dinotrk_profile_classes": (c_int, []),
    "dinotrk_profile_class_name": (c_char_p, [c_int]),
    "dinotrk_profile_enable": (None, [c_int]),
    "dinotrk_profile_collect": (c_int, [POINTER(ctypes.c_double), POINTER(c_ulonglong), c_int]),
    "dinotrk_delta_refine_allgather": (c_int, [_P, c_int, c_int, c_int, POINTER(c_int), POINTER(c_void_p), POINTER(c_void_p), _P,
                                               _P, _P, c_int, c_int, _P, _P, _P, c_size_t, POINTER(c_void_p), c_int, c_size_t, _P]),
    "dinotrk_delta_refine_tc": (c_int, [_P, c_int, c_int, c_int, POINTER(c_int), POINTER(c_void_p), POINTER(c_void_p),
                                        POINTER(c_void_p), _P, _P, _P, c_int, c_int, _P, _P, _P, c_size_t, POINTER(c_void_p),
                                        c_int, c_size_t, _P]),
    "dinotrk_delta_train_saved_bytes": (c_size_t, [c_int, c_int, c_int, POINTER(c_int)]),
    "dinotrk_delta_train_forward_workspace_bytes": (c_size_t, [c_int, c_int, c_int, POINTER(c_int)]),
    "dinotrk_delta_train_backward_workspace_bytes": (c_size_t, [c_int, c_int, c_int, POINTER(c_int)]),
    "dinotrk_delta_train_forward": (c_int, [_P, c_int, c_int, c_int, POINTER(c_int), POINTER(c_void_p), POINTER(c_void_p),
                                            POINTER(c_void_p), POINTER(c_void_p), POINTER(c_void_p), POINTER(c_void_p),
                                            POINTER(c_void_p), c_int, c_float, c_float, _P, _P, c_int, c_int, _P, _P, c_size_t,
                                            _P, c_size_t, _P]),
    "dinotrk_delta_train_backward": (c_int, [_P, c_int, c_int, c_int, POINTER(c_int), POINTER(c_void_p), POINTER(c_void_p),
                                             POINTER(c_void_p), POINTER(c_void_p), c_int, _P, _P, c_int, c_int, _P, _P, c_size_t,
                                             POINTER(c_void_p), POINTER(c_void_p), POINTER(c_void_p), POINTER(c_void_p), _P,
                                             c_size_t, _P]),
    "dinotrk_peer_alloc": (c_int, [c_size_t, POINTER(c_void_p), ctypes.c_char_p]),
    "dinotrk_peer_open": (c_int, [ctypes.c_char_p, POINTER(c_void_p)]),
    "dinotrk_peer_close": (c_int, [_P]),
    "dinotrk_peer_free": (c_int, [_P]),
    "dinotrk_occlusion": (c_int, [_P, _P, _P, c_int, c_int, c_float, c_float, _P, _P]),
    "dinotrk_flow_masks": (c_int, [POINTER(FlowVideo), c_float, _P, _P]),
    "dinotrk_traj_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "dinotrk_traj_chain": (c_int, [POINTER(FlowVideo), _P, c_int, c_float, c_int, _P, _P, c_float, _P, _P, c_size_t, _P]),
    "dinotrk_traj_emit": (c_int, [POINTER(FlowVideo), c_int, _P, _P, c_size_t, _P]),
    "dinotrk_traj_nearest_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "dinotrk_traj_nearest": (c_int, [_P, c_int, c_int, c_int, c_int, c_float, c_float, _P, _P, c_size_t, _P]),
    "dinotrk_of_filter": (c_int, [_P, c_int, c_int, _P, c_int, c_int, c_int, _P, _P, _P, _P, _P, c_int, c_int, _P, _P]),
    "dinotrk_pca_workspace_bytes": (c_size_t, [ctypes.c_longlong, c_int, c_int]),
    "dinotrk_pca_stats": (c_int, [_P, ctypes.c_longlong, c_int, c_int, _P, _P, _P, c_size_t, _P]),
    "dinotrk_pca_power": (c_int, [_P, ctypes.c_longlong, c_int, c_int, _P, _P, _P, _P, _P, _P, c_size_t, _P]),
    "dinotrk_fg_mask": (c_int, [_P, c_int, c_int, c_int, c_int, c_int, _P, _P, c_float, c_int, c_int, _P, _P, _P, _P, c_size_t,
                                _P]),
    "dinotrk_mask_upsample": (c_int, [_P, c_int, c_int, c_int, c_int, c_int, _P, _P]),
    "dinotrk_traj_split_workspace_bytes": (c_size_t, [c_int]),
    "dinotrk_traj_split_count": (c_int, [_P, c_int, c_int, _P, c_int, c_int, c_int, POINTER(c_int), _P, c_size_t, _P]),
    "dinotrk_traj_split_emit": (c_int, [_P, c_int, c_int, _P, _P, _P, c_size_t, _P]),
    "dinotrk_bb_contrastive_cos_stride": (c_int, [c_int]),
    "dinotrk_bb_contrastive_forward_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int, c_int]),
    "dinotrk_bb_contrastive_forward": (c_int, [_P, c_int, c_int, c_int, _P, _P, c_int, _P, _P, _P, _P, c_int, c_float, _P, _P,
                                               _P, c_size_t, _P]),
    "dinotrk_bb_contrastive_backward_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int, _P, _P, _P, _P, c_int]),
    "dinotrk_bb_contrastive_backward": (c_int, [_P, c_int, c_int, c_int, _P, _P, c_int, _P, _P, _P, _P, c_int, c_float, _P, _P,
                                                _P, _P, _P, _P, _P, _P, _P, _P, c_size_t, _P]),
    "dinotrk_sampler_workspace_bytes": (c_size_t, [c_int]),
    "dinotrk_sampler_prepare_count": (c_int, [_P, c_int, c_int, POINTER(c_int), _P, c_size_t, _P]),
    "dinotrk_sampler_prepare_emit": (c_int, [_P, c_int, c_int, _P, _P, _P, c_size_t, _P]),
    "dinotrk_sampler_count": (c_int, [_P, c_int, c_int, _P, c_int, POINTER(c_int), _P, c_size_t, _P]),
    "dinotrk_sampler_select": (c_int, [_P, c_int, c_int, _P, c_int, _P, c_int, _P, _P, _P, c_size_t, _P]),
    "dinotrk_sampler_gather": (c_int, [_P, c_int, _P, _P, c_int, _P, _P, _P]),
    "dinotrk_raft_encode_workspace_bytes": (c_size_t, [c_int, c_int]),
    "dinotrk_raft_encode": (c_int, [_P, c_int, c_int, c_int, c_int, POINTER(RaftWeights), _P, _P, _P, c_size_t, _P]),
    "dinotrk_raft_flow_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "dinotrk_raft_flow": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, c_int, POINTER(c_int), c_int, c_int,
                                  POINTER(RaftWeights), _P, _P, c_size_t, _P]),
}


def lib_path():
    return _build.LIB_PATH


def load(build_if_missing=True):
    """Load (building in-tree if needed) libdinotrk.so.  Raises if that is impossible."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = lib_path()
    if not os.path.exists(path):
        if not build_if_missing:
            raise DinotrkError(f"{path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'`")
        _build.build()
    lib = ctypes.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    if lib.dinotrk_version() < 100:
        raise DinotrkError("libdinotrk.so is older than the Python binding")
    _LIB = lib
    return lib


def check(rc, what="dinotrk"):
    if rc != 0:
        raise DinotrkError(f"{what} failed ({rc}): {load().dinotrk_last_error().decode()}")


def ptr(t):
    if t is None:
        return None
    assert t.is_cuda and t.is_contiguous(), "device pointers must come from contiguous CUDA tensors"
    return c_void_p(t.data_ptr())


def stream_ptr(device=None):
    """Current torch stream of ``device`` (default: the current device).  The library launches on the CURRENT device,
    so callers that own a device wrap their calls in ``torch.cuda.device(dev)`` (see ``on_device``)."""
    return c_void_p(torch.cuda.current_stream(device).cuda_stream)


def on_device(fn):
    """Method decorator: run with ``self._dev`` as the current CUDA device (kernels, streams and the library's
    per-device state then all belong to the model's device, whatever the caller's current device is)."""
    import functools

    @functools.wraps(fn)
    def wrapped(self, *a, **kw):
        with torch.cuda.device(self._dev):
            return fn(self, *a, **kw)
    return wrapped


def require_cuda(device):
    if not torch.cuda.is_available():
        raise DinotrkError("dino_tracker_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
    dev = torch.device(device)
    if dev.type != "cuda":
        raise DinotrkError(f"dino_tracker_b200 runs on CUDA only, got device={device!r}")
    return dev


def make_features(tpc, norms, hi=None, lo=None, quant=None):
    """quant: (q8, fac, rho_f) of quantise_features, or None (the anchor phase's coarse pass then runs on fp16)."""
    f = Features()
    f.tpc, f.norms = tpc.data_ptr(), norms.data_ptr()
    f.hi = hi.data_ptr() if hi is not None else None
    f.lo = lo.data_ptr() if lo is not None else None
    f.T, f.C = tpc.shape[0], tpc.shape[2]
    if quant is not None:
        f.q8, f.q_fac, f.q_rho = (t.data_ptr() for t in quant)
    f._keep = (tpc, norms, hi, lo, quant)  # keep the tensors alive as long as the struct
    return f


def quantise_s8(x, norms, rows_per_group, stream):
    """int8 rows of a [..., C] fp32 tensor for the coarse pass (include/dinotrk.h: dinotrk_quantise_s8): (q int8 [..., C],
    fac [...], rho [...], rho_max [groups of rows_per_group rows])."""
    C = x.shape[-1]
    rows = x.numel() // C
    q = torch.empty(x.shape, device=x.device, dtype=torch.int8)
    fac = torch.empty(x.shape[:-1], device=x.device, dtype=torch.float32)
    rho = torch.empty(x.shape[:-1], device=x.device, dtype=torch.float32)
    rho_max = torch.empty(-(-rows // rows_per_group), device=x.device, dtype=torch.float32)
    check(load().dinotrk_quantise_s8(ptr(x), ptr(norms), rows, C, rows_per_group, ptr(q), ptr(fac), ptr(rho), ptr(rho_max),
                                     stream), "quantise_s8")
    return q, fac, rho, rho_max


def quantise_features(tpc, norms, stream):
    """(q8 [T][P][C], fac [T][P], rho_f [T]) of a [T][P][C] feature video: the int8 operands of the anchor phase's coarse
    pass, or None where that pass cannot run (C not a multiple of 16 or above 1040)."""
    T, P, C = tpc.shape
    if C % 16 or C > 1040:
        return None
    q, fac, _, rho_f = quantise_s8(tpc, norms, P, stream)
    return q, fac, rho_f


def split_range(tpc, norms, stream):
    """(max |x|, smallest non-zero token norm, in the fp16 split's faithful range?) of a [T][P][C] feature video
    (include/dinotrk.h: dinotrk_split_range).  Reads two floats back: syncs the stream."""
    lib = load()
    rng = torch.empty(2, device=tpc.device, dtype=torch.float32)
    check(lib.dinotrk_split_range(ptr(tpc), tpc.numel(), ptr(norms), norms.numel(), ptr(rng), stream), "split_range")
    max_abs, min_norm = rng.tolist()
    return max_abs, min_norm, bool(lib.dinotrk_split_faithful(max_abs, min_norm, tpc.shape[-1]))


def split_fp16(x, stream):
    hi = torch.empty(x.shape, device=x.device, dtype=torch.float16)
    lo = torch.empty(x.shape, device=x.device, dtype=torch.float16)
    check(load().dinotrk_split_fp16(ptr(x), ptr(hi), ptr(lo), x.numel(), stream), "split_fp16")
    return hi, lo


def split_features(tpc, norms, stream):
    """fp16 hi / lo halves of a feature video for the tensor-core contractions, or (None, None) -- the exact-fp32 path,
    with a RuntimeWarning -- when the video lies outside the split's faithful range."""
    max_abs, min_norm, ok = split_range(tpc, norms, stream)
    if not ok:
        warnings.warn(f"feature video outside the fp16 split's faithful range (max |x| = {max_abs:.3g}, smallest token "
                      f"norm = {min_norm:.3g}, C = {tpc.shape[-1]}): its contractions run on the exact-fp32 path",
                      RuntimeWarning, stacklevel=3)
        return None, None
    return split_fp16(tpc, stream)


def make_geom(H, W, patch=14, stride=7, radius=35):
    g = Geom()
    check(load().dinotrk_make_geom(H, W, patch, stride, radius, ctypes.byref(g)), "make_geom")
    return g


def profile_enable(on=True):
    load().dinotrk_profile_enable(1 if on else 0)


def profile_collect():
    """-> {class name: (total ms, launches)} since the previous collect."""
    lib = load()
    n = lib.dinotrk_profile_classes()
    ms = (ctypes.c_double * n)()
    cnt = (c_ulonglong * n)()
    check(lib.dinotrk_profile_collect(ms, cnt, n), "profile_collect")
    return {lib.dinotrk_profile_class_name(i).decode(): (ms[i], int(cnt[i])) for i in range(n) if cnt[i]}


def infer_stats():
    """{anchor-phase maps, finished by the exact-window path, re-done by the full-map path, pipeline, contraction, coarse pass,
    exact-window maps whose descriptor was read in place / gathered} of the last infer."""
    a = (ctypes.c_longlong * 10)()
    check(load().dinotrk_infer_last_stats(a, 10), "infer_last_stats")
    rho_f = struct.unpack("<f", struct.pack("<I", int(a[7])))[0]
    return {"anchor_maps": int(a[0]), "exact_window": int(a[1]), "full_map": int(a[2]), "pipeline": "exact-window" if a[3] else "full-map",
            "full_map_by_certificate": int(a[4]), "contraction": "fp16x3" if a[5] else "fp32",
            "coarse": "int8" if a[6] else "fp16", "coarse_rho_f": rho_f, "desc_in_place": int(a[8]), "desc_gathered": int(a[9])}


def launch_count():
    return int(load().dinotrk_launch_count())
