"""ctypes binding of libyamb200.so (the C ABI declared in include/yamb200.h).

There is no fallback: if the shared library is missing or no CUDA device is present the compute
entry points raise.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# YAMB_LIB_PATH: an alternative build of the same sources (e.g. the -DYAMB_GEMM_TIMERS variant the
# profiling drivers use); the default is the in-tree library __graft_entry__.build() produces
LIB_PATH = os.environ.get("YAMB_LIB_PATH") or os.path.join(_HERE, "libyamb200.so")

ACT_NONE, ACT_RELU, ACT_RELU6, ACT_SWISH, ACT_HSWISH = 0, 1, 2, 3, 4

c_f32p = C.c_void_p  # device pointers are passed as integers


class BnFwd(C.Structure):
    _fields_ = [
        ("partials", C.c_void_p), ("counter", C.c_void_p),
        ("gamma", C.c_void_p), ("beta", C.c_void_p),
        ("eps", C.c_float), ("momentum", C.c_float),
        ("running_mean", C.c_void_p), ("running_var", C.c_void_p),
        ("num_batches_tracked", C.c_void_p),
        ("scale", C.c_void_p), ("shift", C.c_void_p),
        ("mean", C.c_void_p), ("invstd", C.c_void_p),
        ("count", C.c_int64),
    ]


class BnBwd(C.Structure):
    _fields_ = [
        ("partials", C.c_void_p), ("counter", C.c_void_p),
        ("gamma", C.c_void_p), ("mean", C.c_void_p), ("invstd", C.c_void_p),
        ("dgamma", C.c_void_p), ("dbeta", C.c_void_p),
        ("ca", C.c_void_p), ("cb", C.c_void_p), ("cc", C.c_void_p),
        ("count", C.c_int64),
        ("use_batch_stats", C.c_int32),
    ]


class Gemm(C.Structure):
    _fields_ = [
        ("M", C.c_int32), ("N", C.c_int32), ("K", C.c_int32),
        ("a_mn_major", C.c_int32), ("b_mn_major", C.c_int32),
        ("A", C.c_void_p), ("lda", C.c_int64),
        ("B", C.c_void_p), ("ldb", C.c_int64),
        ("D", C.c_void_p), ("ldd", C.c_int64),
        ("epi", C.c_int32),
        ("a_xform", C.c_int32), ("a_act", C.c_int32),
        ("a_scale", C.c_void_p), ("a_shift", C.c_void_p), ("a_scale2", C.c_void_p),
        ("A2", C.c_void_p), ("lda2", C.c_int64),
        ("b_xform", C.c_int32), ("b_act", C.c_int32),
        ("b_scale", C.c_void_p), ("b_shift", C.c_void_p), ("b_scale2", C.c_void_p),
        ("B2", C.c_void_p), ("ldb2", C.c_int64),
        ("residual", C.c_void_p), ("ldr", C.c_int64),
        ("bn_fwd", C.POINTER(BnFwd)),
        ("H", C.c_void_p), ("ldh", C.c_int64),
        ("h_scale", C.c_void_p), ("h_shift", C.c_void_p), ("h_act", C.c_int32),
        ("bn_bwd", C.POINTER(BnBwd)),
        ("max_ctas", C.c_int32),
        ("a_gate", C.c_void_p), ("b_gate", C.c_void_p), ("gate_rows_per_sample", C.c_int64),
    ]


class DwFwd(C.Structure):
    _fields_ = [
        ("N", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("C", C.c_int32),
        ("ldc", C.c_int32), ("k", C.c_int32), ("stride", C.c_int32),
        ("x", C.c_void_p),
        ("in_scale", C.c_void_p), ("in_shift", C.c_void_p), ("in_act", C.c_int32),
        ("w", C.c_void_p), ("y", C.c_void_p),
        ("bn", C.POINTER(BnFwd)),
    ]


class DwBwd(C.Structure):
    _fields_ = [
        ("N", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("C", C.c_int32),
        ("ldc", C.c_int32), ("k", C.c_int32), ("stride", C.c_int32),
        ("dz", C.c_void_p), ("h", C.c_void_p),
        ("ca", C.c_void_p), ("cb", C.c_void_p), ("cc", C.c_void_p),
        ("w", C.c_void_p), ("dw", C.c_void_p),
        ("x", C.c_void_p),
        ("in_scale", C.c_void_p), ("in_shift", C.c_void_p), ("in_act", C.c_int32),
        ("dx", C.c_void_p), ("residual", C.c_void_p),
        ("bn", C.POINTER(BnBwd)),
    ]


class BnApply(C.Structure):
    _fields_ = [
        ("M", C.c_int64), ("C", C.c_int32), ("ldh", C.c_int32), ("ldr", C.c_int32),
        ("ldy", C.c_int32),
        ("h", C.c_void_p), ("scale", C.c_void_p), ("shift", C.c_void_p), ("act", C.c_int32),
        ("residual", C.c_void_p), ("y", C.c_void_p),
        ("gate", C.c_void_p), ("rows_per_sample", C.c_int64),
        ("residual2", C.c_void_p), ("ldr2", C.c_int32),
    ]


class BnReduce(C.Structure):
    _fields_ = [
        ("M", C.c_int64), ("C", C.c_int32), ("lddy", C.c_int32), ("ldh", C.c_int32),
        ("dy", C.c_void_p), ("h", C.c_void_p),
        ("bn", C.POINTER(BnBwd)),
        ("z_scale", C.c_void_p), ("z_shift", C.c_void_p), ("z_act", C.c_int32),
    ]


class BnStats(C.Structure):
    _fields_ = [
        ("M", C.c_int64), ("C", C.c_int32), ("ldh", C.c_int32),
        ("h", C.c_void_p),
        ("bn", C.POINTER(BnFwd)),
    ]


class BnBwdApply(C.Structure):
    _fields_ = [
        ("M", C.c_int64), ("C", C.c_int32), ("lddy", C.c_int32), ("ldh", C.c_int32),
        ("lddh", C.c_int32),
        ("dy", C.c_void_p), ("h", C.c_void_p),
        ("z_scale", C.c_void_p), ("z_shift", C.c_void_p), ("z_act", C.c_int32),
        ("ca", C.c_void_p), ("cb", C.c_void_p), ("cc", C.c_void_p),
        ("dh", C.c_void_p),
    ]


class SePool(C.Structure):
    _fields_ = [
        ("N", C.c_int32), ("HW", C.c_int32), ("C", C.c_int32), ("ldh", C.c_int32),
        ("h", C.c_void_p), ("scale", C.c_void_p), ("shift", C.c_void_p), ("act", C.c_int32),
        ("pooled", C.c_void_p),
    ]


class SeBwdReduce(C.Structure):
    _fields_ = [
        ("N", C.c_int32), ("HW", C.c_int32), ("C", C.c_int32), ("ldd", C.c_int32),
        ("ldh", C.c_int32),
        ("dy", C.c_void_p), ("h", C.c_void_p), ("scale", C.c_void_p), ("shift", C.c_void_p),
        ("act", C.c_int32),
        ("dgate", C.c_void_p),
    ]


class SeBwdApply(C.Structure):
    _fields_ = [
        ("M", C.c_int64), ("C", C.c_int32), ("ldd", C.c_int32), ("ldh", C.c_int32),
        ("ldz", C.c_int32), ("rows_per_sample", C.c_int64),
        ("dy", C.c_void_p), ("h", C.c_void_p), ("scale", C.c_void_p), ("shift", C.c_void_p),
        ("act", C.c_int32),
        ("gate", C.c_void_p), ("dpool", C.c_void_p), ("ldg", C.c_int32), ("dz", C.c_void_p),
        ("bn", C.POINTER(BnBwd)),
    ]


class Rmsprop(C.Structure):
    _fields_ = [
        ("n", C.c_int64),
        ("p", C.c_void_p), ("g", C.c_void_p), ("sq", C.c_void_p), ("mom", C.c_void_p),
        ("grad_avg", C.c_void_p),
        ("ema", C.c_void_p), ("p_bf16", C.c_void_p), ("wd_mask", C.c_void_p),
        ("hyper", C.c_void_p),
        ("lr", C.c_float), ("alpha", C.c_float), ("eps", C.c_float), ("momentum", C.c_float),
        ("weight_decay", C.c_float), ("l2", C.c_float), ("grad_scale", C.c_float),
        ("ema_m", C.c_float),
        ("eps_inside_sqrt", C.c_int32), ("centered", C.c_int32),
    ]


class Sgd(C.Structure):
    _fields_ = [
        ("n", C.c_int64),
        ("p", C.c_void_p), ("g", C.c_void_p), ("mom", C.c_void_p),
        ("ema", C.c_void_p), ("p_bf16", C.c_void_p), ("wd_mask", C.c_void_p),
        ("hyper", C.c_void_p),
        ("lr", C.c_float), ("momentum", C.c_float), ("dampening", C.c_float),
        ("weight_decay", C.c_float), ("l2", C.c_float), ("grad_scale", C.c_float),
        ("ema_m", C.c_float),
        ("nesterov", C.c_int32),
    ]


class SeFc(C.Structure):
    _fields_ = [
        ("N", C.c_int32), ("C", C.c_int32), ("R", C.c_int32), ("act", C.c_int32),
        ("pooled", C.c_void_p),
        ("w_r", C.c_void_p), ("b_r", C.c_void_p), ("w_e", C.c_void_p), ("b_e", C.c_void_p),
        ("u", C.c_void_p), ("v", C.c_void_p), ("gate", C.c_void_p),
    ]


class SeFcBwd(C.Structure):
    _fields_ = [
        ("N", C.c_int32), ("C", C.c_int32), ("R", C.c_int32), ("act", C.c_int32),
        ("inv_hw", C.c_float),
        ("dgate", C.c_void_p), ("gate", C.c_void_p), ("u", C.c_void_p), ("v", C.c_void_p),
        ("pooled", C.c_void_p), ("w_r", C.c_void_p), ("w_e", C.c_void_p),
        ("dpool", C.c_void_p), ("dt", C.c_void_p), ("du", C.c_void_p),
        ("g_wr", C.c_void_p), ("g_br", C.c_void_p), ("g_we", C.c_void_p), ("g_be", C.c_void_p),
    ]


class SoftmaxCe(C.Structure):
    _fields_ = [
        ("N", C.c_int32), ("C", C.c_int32), ("ld", C.c_int64),
        ("logits", C.c_void_p), ("target", C.c_void_p),
        ("smoothing", C.c_float),
        ("loss", C.c_void_p), ("correct1", C.c_void_p), ("correct5", C.c_void_p),
        ("G", C.c_void_p), ("ldg", C.c_int64),
    ]


class SoftmaxCeGrad(C.Structure):
    _fields_ = [
        ("N", C.c_int32), ("C", C.c_int32),
        ("G", C.c_void_p), ("ldg", C.c_int64),
        ("dloss", C.c_void_p),
        ("dlogits", C.c_void_p), ("ldd", C.c_int64),
        ("dbias", C.c_void_p),
    ]


class StemConv(C.Structure):
    _fields_ = [
        ("N", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("Cout", C.c_int32),
        ("x", C.c_void_p), ("w", C.c_void_p), ("y", C.c_void_p),
        ("dh", C.c_void_p), ("dw", C.c_void_p),
    ]


class BnEval(C.Structure):
    _fields_ = [
        ("gamma", C.c_void_p), ("beta", C.c_void_p),
        ("running_mean", C.c_void_p), ("running_var", C.c_void_p),
        ("eps", C.c_float),
    ]


class BlockEval(C.Structure):
    _fields_ = [
        ("N", C.c_int32), ("H", C.c_int32), ("W", C.c_int32),
        ("Cin", C.c_int32), ("Chid", C.c_int32), ("Cout", C.c_int32),
        ("kernel", C.c_int32), ("stride", C.c_int32),
        ("act", C.c_int32), ("residual", C.c_int32),
        ("x", C.c_void_p), ("w_expand", C.c_void_p), ("w_dw", C.c_void_p),
        ("w_project", C.c_void_p),
        ("bn1", BnEval), ("bn2", BnEval), ("bn3", BnEval),
        ("y", C.c_void_p),
        ("gate", C.c_void_p), ("pooled", C.c_void_p),
    ]


class NlGram(C.Structure):
    _fields_ = [
        ("N", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("sub", C.c_int32),
        ("X", C.c_void_p), ("ldx", C.c_int64), ("I", C.c_int32),
        ("Y", C.c_void_p), ("ldy", C.c_int64), ("J", C.c_int32),
        ("alpha", C.c_float),
        ("G", C.c_void_p),
    ]


class NlRowmat(C.Structure):
    _fields_ = [
        ("N", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("sub", C.c_int32),
        ("X", C.c_void_p), ("ldx", C.c_int64), ("K", C.c_int32),
        ("Mat", C.c_void_p), ("mat_stride", C.c_int64), ("sk", C.c_int64), ("so", C.c_int64),
        ("O", C.c_int32),
        ("alpha", C.c_float),
        ("base", C.c_void_p), ("ldb", C.c_int64), ("O_copy", C.c_int32),
        ("accumulate", C.c_int32),
        ("out", C.c_void_p), ("ldo", C.c_int64),
    ]


class InFwd(C.Structure):
    _fields_ = [
        ("N", C.c_int32), ("HW", C.c_int32), ("C", C.c_int32), ("ldh", C.c_int32),
        ("h", C.c_void_p),
        ("gamma", C.c_void_p), ("beta", C.c_void_p),
        ("eps", C.c_float), ("momentum", C.c_float),
        ("running_mean", C.c_void_p), ("running_var", C.c_void_p),
        ("mean", C.c_void_p), ("invstd", C.c_void_p),
        ("residual", C.c_void_p), ("ldr", C.c_int32),
        ("residual2", C.c_void_p), ("ldr2", C.c_int32),
        ("y", C.c_void_p), ("ldy", C.c_int32),
        ("counter", C.c_void_p),
    ]


class InBwd(C.Structure):
    _fields_ = [
        ("N", C.c_int32), ("HW", C.c_int32), ("C", C.c_int32), ("ldh", C.c_int32),
        ("lddy", C.c_int32), ("lddh", C.c_int32),
        ("dy", C.c_void_p), ("h", C.c_void_p),
        ("gamma", C.c_void_p), ("mean", C.c_void_p), ("invstd", C.c_void_p),
        ("dgamma", C.c_void_p), ("dbeta", C.c_void_p),
        ("dh", C.c_void_p),
        ("counter", C.c_void_p),
    ]


_STRUCTS = {0: BnFwd, 1: BnBwd, 2: Gemm, 3: DwFwd, 4: DwBwd, 5: BnApply, 6: BnReduce, 7: SePool,
            8: Rmsprop, 9: SeBwdReduce, 10: SeBwdApply, 11: BnStats, 12: BnBwdApply, 13: NlGram,
            14: NlRowmat, 15: SeFc, 16: SeFcBwd, 17: SoftmaxCe, 18: SoftmaxCeGrad,
            19: StemConv, 20: BnEval, 21: BlockEval, 22: InFwd, 23: InBwd, 24: Sgd}

# every symbol include/yamb200.h declares
SYMBOLS = ["yamb_pointwise_gemm", "yamb_depthwise_fwd", "yamb_depthwise_bwd", "yamb_bn_apply_fwd",
           "yamb_bn_reduce_bwd", "yamb_bn_stats_fwd", "yamb_bn_bwd_apply_bwd", "yamb_se_pool_fwd", "yamb_se_bwd_reduce_bwd", "yamb_se_bwd_apply_bwd", "yamb_nl_gram_fwd", "yamb_nl_rowmat_fwd", "yamb_se_fc_fwd", "yamb_se_fc_bwd", "yamb_softmax_ce_fwd", "yamb_softmax_ce_bwd", "yamb_colsum_bf16", "yamb_stem_conv_fwd", "yamb_stem_conv_wgrad", "yamb_block_eval_fwd", "yamb_block_eval_pool_fwd", "yamb_instance_norm_fwd", "yamb_instance_norm_bwd", "yamb_rmsprop_step", "yamb_sgd_step", "yamb_ema_update",
           "yamb_cast_bf16", "yamb_max_ctas", "yamb_struct_size", "yamb_last_error",
           "yamb_version"]
_lib = None


class NativeError(RuntimeError):
    pass


def lib():
    """Load libyamb200.so (once). Raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise NativeError(
                "libyamb200.so not built: run `python -c 'import __graft_entry__ as g; g.build()'`")
        l = C.CDLL(LIB_PATH)
        l.yamb_last_error.restype = C.c_char_p
        l.yamb_struct_size.argtypes = [C.c_int]
        for which, st in _STRUCTS.items():
            n = l.yamb_struct_size(which)
            if n != C.sizeof(st):
                raise NativeError("ABI mismatch for struct %d: C %d vs ctypes %d" %
                                  (which, n, C.sizeof(st)))
        l.yamb_pointwise_gemm.argtypes = [C.POINTER(Gemm), C.c_void_p]
        l.yamb_depthwise_fwd.argtypes = [C.POINTER(DwFwd), C.c_void_p]
        l.yamb_depthwise_bwd.argtypes = [C.POINTER(DwBwd), C.c_void_p]
        l.yamb_bn_apply_fwd.argtypes = [C.POINTER(BnApply), C.c_void_p]
        l.yamb_bn_reduce_bwd.argtypes = [C.POINTER(BnReduce), C.c_void_p]
        l.yamb_bn_stats_fwd.argtypes = [C.POINTER(BnStats), C.c_void_p]
        l.yamb_bn_bwd_apply_bwd.argtypes = [C.POINTER(BnBwdApply), C.c_void_p]
        l.yamb_se_pool_fwd.argtypes = [C.POINTER(SePool), C.c_void_p]
        l.yamb_se_bwd_reduce_bwd.argtypes = [C.POINTER(SeBwdReduce), C.c_void_p]
        l.yamb_se_bwd_apply_bwd.argtypes = [C.POINTER(SeBwdApply), C.c_void_p]
        l.yamb_softmax_ce_fwd.argtypes = [C.POINTER(SoftmaxCe), C.c_void_p]
        l.yamb_softmax_ce_bwd.argtypes = [C.POINTER(SoftmaxCeGrad), C.c_void_p]
        l.yamb_colsum_bf16.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_int64, C.c_void_p,
                                       C.c_void_p]
        l.yamb_stem_conv_fwd.argtypes = [C.POINTER(StemConv), C.c_void_p]
        l.yamb_stem_conv_wgrad.argtypes = [C.POINTER(StemConv), C.c_void_p]
        l.yamb_se_fc_fwd.argtypes = [C.POINTER(SeFc), C.c_void_p]
        l.yamb_se_fc_bwd.argtypes = [C.POINTER(SeFcBwd), C.c_void_p]
        l.yamb_nl_gram_fwd.argtypes = [C.POINTER(NlGram), C.c_void_p]
        l.yamb_nl_rowmat_fwd.argtypes = [C.POINTER(NlRowmat), C.c_void_p]
        l.yamb_block_eval_fwd.argtypes = [C.POINTER(BlockEval), C.c_void_p]
        l.yamb_block_eval_pool_fwd.argtypes = [C.POINTER(BlockEval), C.c_void_p]
        l.yamb_instance_norm_fwd.argtypes = [C.POINTER(InFwd), C.c_void_p]
        l.yamb_instance_norm_bwd.argtypes = [C.POINTER(InBwd), C.c_void_p]
        l.yamb_rmsprop_step.argtypes = [C.POINTER(Rmsprop), C.c_void_p]
        l.yamb_sgd_step.argtypes = [C.POINTER(Sgd), C.c_void_p]
        l.yamb_ema_update.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_float,
                                      C.c_void_p]
        l.yamb_cast_bf16.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
        _lib = l
    return _lib


def check(rc):
    if rc != 0:
        raise NativeError("yamb200 error %d: %s" % (rc, lib().yamb_last_error().decode()))


def ptr(t):
    """Device pointer of a torch tensor (None -> NULL)."""
    return None if t is None else t.data_ptr()


def stream_handle():
    import torch
    return torch.cuda.current_stream().cuda_stream
