"""ctypes binding of libcoclr_b200.so (include/coclr_b200.h).

There is no CPU path: importing is cheap, but every op raises if the CUDA library is missing or
the tensors are not on a CUDA device.  PyTorch is used only for device memory and streams.
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libcoclr_b200.so")
_lib = None


class CoclrError(RuntimeError):
    pass


class Src(C.Structure):
    _fields_ = [("hi", C.c_void_p), ("lo", C.c_void_p), ("ld", C.c_int), ("coff", C.c_int), ("C", C.c_int),
                ("T", C.c_int), ("H", C.c_int), ("W", C.c_int)]


class Geom(C.Structure):
    _fields_ = [("kt", C.c_int), ("kh", C.c_int), ("kw", C.c_int),
                ("st", C.c_int), ("sh", C.c_int), ("sw", C.c_int),
                ("pt", C.c_int), ("ph", C.c_int), ("pw", C.c_int),
                ("transposed", C.c_int)]


class Conv(C.Structure):
    _fields_ = [("src", Src), ("g", Geom),
                ("B", C.c_int), ("Td", C.c_int), ("Hd", C.c_int), ("Wd", C.c_int),
                ("Kreal", C.c_int), ("wpk", C.c_void_p), ("wunscale", C.c_void_p),
                ("N", C.c_int), ("BN", C.c_int), ("n_tiles", C.c_int),
                ("dst", C.c_void_p), ("dst_ld", C.c_int), ("dst_coff", C.c_int),
                ("accumulate", C.c_int), ("stats_sum", C.c_void_p), ("stats_sq", C.c_void_p),
                ("npass", C.c_int), ("a_bf16", C.c_int), ("b_bf16", C.c_int), ("out_scale", C.c_void_p)]


class Wgrad(C.Structure):
    _fields_ = [("src", Src), ("g", Geom), ("dy", Src),
                ("B", C.c_int), ("Td", C.c_int), ("Hd", C.c_int), ("Wd", C.c_int),
                ("Cout", C.c_int), ("Cin_real", C.c_int), ("dw", C.c_void_p),
                ("npass", C.c_int), ("dy_bf16", C.c_int), ("src_bf16", C.c_int), ("splits", C.c_int),
                ("out_scale", C.c_void_p), ("ws", C.c_void_p), ("ws_floats", C.c_long)]


class Pack(C.Structure):
    _fields_ = [("w", C.c_void_p), ("Cout", C.c_int), ("Cin", C.c_int), ("taps", C.c_int),
                ("Cpad", C.c_int), ("mode", C.c_int), ("bf16", C.c_int),
                ("wpk", C.c_void_p), ("unscale", C.c_void_p)]


class BnFinalize(C.Structure):
    _fields_ = [("sum", C.c_void_p), ("sumsq", C.c_void_p), ("count", C.c_long),
                ("gamma", C.c_void_p), ("beta", C.c_void_p),
                ("running_mean", C.c_void_p), ("running_var", C.c_void_p),
                ("momentum", C.c_float), ("eps", C.c_float), ("training", C.c_int),
                ("scale", C.c_void_p), ("shift", C.c_void_p),
                ("save_mean", C.c_void_p), ("save_rstd", C.c_void_p), ("C", C.c_int)]


class Split(C.Structure):
    _fields_ = [("x", C.c_void_p), ("ld", C.c_int), ("coff", C.c_int), ("C", C.c_int), ("M", C.c_long),
                ("scale", C.c_void_p), ("shift", C.c_void_p), ("relu", C.c_int),
                ("hi", C.c_void_p), ("lo", C.c_void_p), ("out_ld", C.c_int), ("out_coff", C.c_int),
                ("bf16", C.c_int), ("hi2", C.c_void_p), ("lo2", C.c_void_p), ("bn", BnFinalize),
                ("res_hi", C.c_void_p), ("res_lo", C.c_void_p), ("res_ld", C.c_int), ("res_coff", C.c_int)]


class BnBwd(C.Structure):
    _fields_ = [("y", C.c_void_p), ("dA", C.c_void_p), ("ld", C.c_int), ("coff", C.c_int), ("C", C.c_int),
                ("M", C.c_long), ("scale", C.c_void_p), ("shift", C.c_void_p),
                ("mean", C.c_void_p), ("rstd", C.c_void_p), ("relu", C.c_int),
                ("sums", C.c_void_p), ("dgamma", C.c_void_p), ("dbeta", C.c_void_p),
                ("dy_hi", C.c_void_p), ("dy_lo", C.c_void_p),
                ("res_hi", C.c_void_p), ("res_lo", C.c_void_p), ("res_ld", C.c_int), ("res_coff", C.c_int),
                ("res_bf16", C.c_int), ("dres", C.c_void_p), ("dres_ld", C.c_int), ("dres_coff", C.c_int),
                ("dres_accumulate", C.c_int), ("dy_fp16", C.c_int), ("amax", C.c_void_p), ("dy_scale", C.c_void_p)]


class Pool(C.Structure):
    _fields_ = [("x_hi", C.c_void_p), ("x_lo", C.c_void_p), ("ldx", C.c_int), ("x_coff", C.c_int),
                ("y_hi", C.c_void_p), ("y_lo", C.c_void_p), ("ldy", C.c_int), ("y_coff", C.c_int),
                ("y2_hi", C.c_void_p), ("y2_lo", C.c_void_p), ("idx", C.c_void_p),
                ("B", C.c_int), ("C", C.c_int), ("Ti", C.c_int), ("Hi", C.c_int), ("Wi", C.c_int),
                ("To", C.c_int), ("Ho", C.c_int), ("Wo", C.c_int), ("g", Geom),
                ("dy", C.c_void_p), ("dx", C.c_void_p), ("accumulate", C.c_int),
                ("y", C.c_void_p), ("scale", C.c_void_p), ("shift", C.c_void_p), ("relu", C.c_int)]


class Adam(C.Structure):
    _fields_ = [("param", C.c_void_p), ("grad", C.c_void_p), ("exp_avg", C.c_void_p), ("exp_avg_sq", C.c_void_p),
                ("n", C.c_long), ("grad_scale", C.c_float),
                ("beta1", C.c_float), ("beta2", C.c_float), ("eps", C.c_float), ("weight_decay", C.c_float),
                ("step_size", C.c_float), ("bc2_sqrt", C.c_float)]


class Sgd(C.Structure):
    _fields_ = [("param", C.c_void_p), ("grad", C.c_void_p), ("momentum_buf", C.c_void_p), ("n", C.c_long),
                ("lr", C.c_float), ("weight_decay", C.c_float), ("momentum", C.c_float), ("first", C.c_int)]


class ClsHead(C.Structure):
    _fields_ = [("B", C.c_int), ("fs", C.c_int), ("ncls", C.c_int),
                ("l2norm", C.c_int), ("bn", C.c_int), ("bn_training", C.c_int), ("dropout", C.c_int),
                ("p", C.c_float), ("momentum", C.c_float), ("eps", C.c_float),
                ("seed", C.c_ulonglong), ("offset", C.c_ulonglong),
                ("feat", C.c_void_p), ("xn", C.c_void_p), ("inv_norm", C.c_void_p),
                ("xb", C.c_void_p), ("mean", C.c_void_p), ("rstd", C.c_void_p),
                ("gamma", C.c_void_p), ("beta", C.c_void_p), ("running_mean", C.c_void_p), ("running_var", C.c_void_p),
                ("mask", C.c_void_p), ("xd", C.c_void_p),
                ("W", C.c_void_p), ("bias", C.c_void_p), ("logits", C.c_void_p),
                ("dlogits", C.c_void_p), ("dW", C.c_void_p), ("dbias", C.c_void_p), ("dgamma", C.c_void_p),
                ("dbeta", C.c_void_p), ("dx", C.c_void_p), ("dfeat", C.c_void_p)]


class VideoFinalize(C.Structure):
    _fields_ = [("prob_sum", C.c_void_p), ("feat_sum", C.c_void_p), ("count", C.c_void_p),
                ("Nv", C.c_int), ("C", C.c_int), ("D", C.c_int), ("n_views", C.c_int),
                ("feat_mean", C.c_void_p), ("prob_mean", C.c_void_p), ("views_sum", C.c_void_p), ("prob", C.c_void_p),
                ("target", C.c_void_p), ("rank", C.c_void_p), ("hits", C.c_void_p)]


class Probe(C.Structure):
    _fields_ = [("N", C.c_int), ("Nq", C.c_int), ("D", C.c_int), ("C", C.c_int), ("S", C.c_int),
                ("epochs", C.c_int), ("batch", C.c_int), ("eval_freq", C.c_int), ("final_bn", C.c_int),
                ("momentum", C.c_float), ("eps", C.c_float),
                ("train", C.c_void_p), ("train_label", C.c_void_p), ("test", C.c_void_p), ("test_label", C.c_void_p),
                ("order", C.c_void_p), ("lr", C.c_void_p), ("wd", C.c_void_p),
                ("W", C.c_void_p), ("bias", C.c_void_p), ("gamma", C.c_void_p), ("beta", C.c_void_p),
                ("W_buf", C.c_void_p), ("bias_buf", C.c_void_p), ("gamma_buf", C.c_void_p), ("beta_buf", C.c_void_p),
                ("running_mean", C.c_void_p), ("running_var", C.c_void_p), ("work", C.c_void_p),
                ("train_loss", C.c_void_p), ("train_hits", C.c_void_p), ("val_loss", C.c_void_p),
                ("val_hits", C.c_void_p), ("prob", C.c_void_p)]


class Augment(C.Structure):
    _fields_ = [("src", C.c_void_p), ("B", C.c_int), ("F", C.c_int), ("Hmax", C.c_int), ("Wmax", C.c_int),
                ("S", C.c_int), ("D", C.c_int), ("K", C.c_int), ("band_rows", C.c_int),
                ("clips", C.c_void_p), ("coef", C.c_void_p), ("bounds", C.c_void_p), ("gray", C.c_void_p),
                ("out", C.c_void_p), ("out_batch_stride", C.c_long), ("out_clip_stride", C.c_long),
                ("out_chan_stride", C.c_long)]


class AugmentClf(C.Structure):
    _fields_ = [("src", C.c_void_p), ("NF", C.c_int), ("Hmax", C.c_int), ("Wmax", C.c_int), ("n_frames", C.c_int),
                ("frames", C.c_void_p), ("samples", C.c_void_p),
                ("M", C.c_int), ("D", C.c_int), ("K1", C.c_int), ("K2", C.c_int), ("band_rows", C.c_int),
                ("rows", C.c_int), ("coef1", C.c_void_p), ("bounds1", C.c_void_p), ("coef2", C.c_void_p),
                ("bounds2", C.c_void_p), ("out", C.c_void_p)]


class Jpeg(C.Structure):
    _fields_ = [("n", C.c_int), ("data", C.c_void_p), ("frames", C.c_void_p), ("frames_host", C.c_void_p),
                ("quant", C.c_void_p), ("huff", C.c_void_p), ("out", C.c_void_p),
                ("frame_stride", C.c_int64), ("row_stride", C.c_int64), ("status", C.c_void_p),
                ("work", C.c_void_p), ("work_bytes", C.c_size_t)]


class JpegEncode(C.Structure):
    _fields_ = [("n", C.c_int), ("h", C.c_int), ("w", C.c_int), ("quality", C.c_int), ("subsampling", C.c_int),
                ("rgb", C.c_void_p), ("frame_stride", C.c_int64), ("row_stride", C.c_int64),
                ("out", C.c_void_p), ("out_bytes", C.c_size_t), ("offsets", C.c_void_p),
                ("work", C.c_void_p), ("work_bytes", C.c_size_t)]


class Tvl1(C.Structure):
    _fields_ = [("P", C.c_int), ("H", C.c_int), ("W", C.c_int), ("i0", C.c_void_p), ("i1", C.c_void_p),
                ("flow", C.c_void_p), ("iterations", C.c_void_p), ("work", C.c_void_p), ("work_bytes", C.c_size_t)]


class JpegSlots(C.Structure):
    _fields_ = [("slot_begin", C.c_void_p), ("slots", C.c_void_p), ("slot_begin_host", C.c_void_p),
                ("slots_host", C.c_void_p), ("n_out", C.c_int)]


def library_path():
    return _LIB_PATH


def load():
    """Load the CUDA library; raises CoclrError when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        raise CoclrError(
            "libcoclr_b200.so is missing (%s). Build it with `python -m coclr_b200.build` "
            "(needs nvcc with sm_90a support). There is no CPU fallback." % _LIB_PATH)
    lib = C.CDLL(_LIB_PATH)
    from . import _signatures
    _signatures.declare(lib)
    _lib = lib
    return lib


LAUNCHES = 0  # kernels of this library launched so far in this process (bench.py reports the per-step count)
KERNELS_PER_CALL = {"coclr_bn_bwd": 2, "coclr_l2norm_bwd": 2, "coclr_conv_packed_bytes": 0, "coclr_gate_fc_bwd": 2, "coclr_wgrad_ws_floats": 0, "coclr_wgrad_tma_plan": 0,
                    "coclr_center_normalize": 2,
                    "coclr_augment_smem_bytes": 0, "coclr_augment_clf_smem_bytes": 0,
                    "coclr_jpeg_parse": 0, "coclr_jpeg_work_bytes": 0, "coclr_jpeg_decode": 3,
                    "coclr_jpeg_decode_slots": 3, "coclr_jpeg_encode_header": 0,
                    "coclr_jpeg_encode_max_bytes": 0, "coclr_jpeg_encode_work_bytes": 0,
                    "coclr_jpeg_encode": 8,     # per pass: a batch split by its workspace counts one pass
                    "coclr_tvl1_scales": 0, "coclr_tvl1_work_bytes": 0,
                    "coclr_flow_zoom_out": 3, "coclr_flow_warp": 2, "coclr_flow_iterate_work_bytes": 0,
                    # data-dependent (two launches per primal-dual iteration until the pairs converge): not counted
                    "coclr_tvl1": 0, "coclr_flow_iterate": 0}


def kernels_of(fn, args=()):
    """Kernels fn(*args) launches (bench.py reports the per-step total); fn: a library function or its name.  A weight
    gradient (args[0]: its coclr_wgrad_t) on the TMA-staged kernel (a shape it takes, with a large enough workspace) is
    two launches: partial sums, then the reduction over the pixel splits; so is the engine's space-to-depth stem op."""
    name = fn if isinstance(fn, str) else fn.__name__
    if name in ("coclr_conv_wgrad", "coclr_conv_wgrad_s2d") and args:
        wg = args[0]._obj
        if wg.ws and 0 < load().coclr_wgrad_ws_floats(args[0]) <= wg.ws_floats:
            return 2
    return KERNELS_PER_CALL.get(name, 1)


def check(rc, what, args=()):
    global LAUNCHES
    if rc != 0:
        raise CoclrError("%s failed with code %d" % (what, rc))
    LAUNCHES += kernels_of(what, args)


def stream_ptr():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


DRY_RUN = False  # tests only: lets launch plans be BUILT (never run) over CPU tensors to validate their structure


def dptr(t):
    if t is None:
        return None
    if not t.is_cuda and not DRY_RUN:
        raise CoclrError("coclr_b200 ops need CUDA tensors (no CPU fallback)")
    return C.c_void_p(t.data_ptr())


_num_sms = {}


def num_sms(device=None):
    if DRY_RUN:
        return 132   # H100 SXM
    dev = torch.cuda.current_device() if device is None else torch.device(device).index
    if dev not in _num_sms:
        _num_sms[dev] = torch.cuda.get_device_properties(dev).multi_processor_count
    return _num_sms[dev]
