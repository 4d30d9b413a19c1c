"""ctypes binding of libddnm_b200.so (include/ddnm_b200.h).  There is NO fallback: if the CUDA library is
missing or fails to load, importing the product path raises."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libddnm_b200.so")


class DDNMError(RuntimeError):
    pass


class SimpleCfg(C.Structure):
    _fields_ = [("ch", C.c_int), ("out_ch", C.c_int), ("n_levels", C.c_int), ("ch_mult", C.c_int * 8),
                ("num_res_blocks", C.c_int), ("n_attn_res", C.c_int), ("attn_res", C.c_int * 4),
                ("in_channels", C.c_int), ("resolution", C.c_int), ("groups", C.c_int), ("eps", C.c_float)]


class OpenAICfg(C.Structure):
    _fields_ = [("image_size", C.c_int), ("model_channels", C.c_int), ("num_res_blocks", C.c_int), ("n_levels", C.c_int),
                ("channel_mult", C.c_int * 8), ("n_attn_ds", C.c_int), ("attn_ds", C.c_int * 4),
                ("num_head_channels", C.c_int), ("out_channels", C.c_int), ("in_channels", C.c_int), ("groups", C.c_int),
                ("eps", C.c_float), ("num_classes", C.c_int)]


class ClassifierCfg(C.Structure):
    _fields_ = [("image_size", C.c_int), ("model_channels", C.c_int), ("num_res_blocks", C.c_int), ("n_levels", C.c_int),
                ("channel_mult", C.c_int * 8), ("n_attn_ds", C.c_int), ("attn_ds", C.c_int * 4),
                ("num_head_channels", C.c_int), ("out_channels", C.c_int), ("in_channels", C.c_int), ("groups", C.c_int),
                ("eps", C.c_float), ("pool", C.c_int)]


class ClassifierGuidance(C.Structure):
    _fields_ = [("classifier", C.c_void_p), ("x", C.c_void_p), ("labels", C.c_void_p), ("scale", C.c_float),
                ("grad_buf", C.c_void_p), ("batch", C.c_int), ("labels_checked", C.c_int)]


class OperatorDesc(C.Structure):
    _fields_ = [("kind", C.c_int), ("channels", C.c_int), ("img_dim", C.c_int), ("ratio", C.c_int),
                ("v_small", C.c_void_p), ("u_small", C.c_void_p), ("singulars", C.c_void_p),
                ("singulars_orig", C.c_void_p), ("perm", C.c_void_p), ("mask", C.c_void_p), ("v_small2", C.c_void_p),
                ("u_small2", C.c_void_p)]


class SimpleDeg(C.Structure):
    _fields_ = [("use_mask", C.c_int), ("use_gray", C.c_int), ("scale", C.c_int), ("img_dim", C.c_int), ("channels", C.c_int),
                ("mask", C.c_void_p)]


class HqScalars(C.Structure):
    _fields_ = [("c_recip", C.c_float), ("c_recipm1", C.c_float), ("coef1", C.c_float), ("coef2", C.c_float), ("lambda_t", C.c_float),
                ("gamma_t", C.c_float), ("nonzero", C.c_float), ("clip", C.c_int)]


class Schedule(C.Structure):
    _fields_ = [("n_pairs", C.c_int), ("t_i", C.c_void_p), ("t_j", C.c_void_p), ("abar", C.c_void_p),
                ("num_timesteps", C.c_int), ("eta", C.c_float), ("sigma_y", C.c_float), ("plus", C.c_int)]


_lib = None

_P, _I, _LL, _F, _D = C.c_void_p, C.c_int, C.c_longlong, C.c_float, C.c_double
# classifier-guidance callback of ddnm_sample_guided: (user, pair_index, t, stream) -> 0 on success
GuidanceFn = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p)

_SIGS = {
    "ddnm_version": (C.c_int, []),
    "ddnm_unet_simple_create": (C.c_int, [C.POINTER(SimpleCfg), _I, C.POINTER(_P)]),
    "ddnm_unet_openai_create": (C.c_int, [C.POINTER(OpenAICfg), _I, C.POINTER(_P)]),
    "ddnm_classifier_create": (C.c_int, [C.POINTER(ClassifierCfg), _I, C.POINTER(_P)]),
    "ddnm_classifier_forward": (C.c_int, [_P, _P, _P, _P, _P]),
    "ddnm_classifier_grad": (C.c_int, [_P, _P, _P, _P, _F, _P, _P, _P]),
    "ddnm_classifier_guidance_fn": (C.c_int, [_P, _I, _I, _P]),
    "ddnm_unet_set_param": (C.c_int, [_P, C.c_char_p, _P, _LL]),
    "ddnm_unet_set_precision": (C.c_int, [_P, _I]),
    "ddnm_unet_finalize": (C.c_int, [_P]),
    "ddnm_unet_forward": (C.c_int, [_P, _P, _P, _P, _P]),
    "ddnm_unet_forward_cond": (C.c_int, [_P, _P, _P, _P, _P, _P]),
    "ddnm_unet_set_graph": (C.c_int, [_P, _I]),
    "ddnm_unet_read_tap": (C.c_int, [_P, C.c_char_p, _P, _LL, _P]),
    "ddnm_unet_info": (C.c_int, [_P, C.POINTER(_LL), C.POINTER(_I), C.POINTER(_D)]),
    "ddnm_unet_profile": (C.c_int, [_P, _P, _P, _P, _P, C.c_char_p, _LL]),
    "ddnm_unet_destroy": (C.c_int, [_P]),
    "ddnm_operator_create": (C.c_int, [C.POINTER(OperatorDesc), C.POINTER(_P)]),
    "ddnm_operator_y_dim": (_LL, [_P]),
    "ddnm_operator_A": (C.c_int, [_P, _P, _I, _P, _P]),
    "ddnm_operator_A_pinv": (C.c_int, [_P, _P, _I, _P, _P]),
    "ddnm_operator_project": (C.c_int, [_P, _P, _P, _I, _P, _P]),
    "ddnm_operator_lambda": (C.c_int, [_P, _P, _I, _F, _F, _F, _F, _P, _P]),
    "ddnm_operator_lambda_noise": (C.c_int, [_P, _P, _P, _I, _F, _F, _F, _F, _P, _P]),
    "ddnm_operator_destroy": (C.c_int, [_P]),
    "ddnm_sample": (C.c_int, [_P, _P, C.POINTER(Schedule), _P, _P, _P, _I, _P, _P, _P]),
    "ddnm_sample_guided": (C.c_int, [_P, _P, C.POINTER(Schedule), _P, _P, _P, _I, _P, _P, GuidanceFn, _P, _P, _P, _P]),
    "ddnm_sample_range": (C.c_int, [_P, _P, C.POINTER(Schedule), _I, _I, _P, _P, C.POINTER(C.c_int), _P, _P, _I, _P, _P, _P, _P, _P]),
    "ddnm_sample_simplified_range": (C.c_int, [_P, C.POINTER(SimpleDeg), C.POINTER(Schedule), _I, _I, _P, _P, C.POINTER(C.c_int), _P, _P,
                                               _I, _P]),
    "ddnm_simplified_A": (C.c_int, [C.POINTER(SimpleDeg), _P, _I, _P, _P]),
    "ddnm_simplified_Ap": (C.c_int, [C.POINTER(SimpleDeg), _P, _I, _P, _P]),
    "ddnm_sample_simplified": (C.c_int, [_P, C.POINTER(SimpleDeg), C.POINTER(Schedule), _P, _P, _P, _I, _P, _P, _P]),
    "ddnm_hq_canvas": (C.c_int, [_P, _I, _I, _I, _I, _I, _P, _P]),
    "ddnm_hq_step": (C.c_int, [C.POINTER(SimpleDeg), _P, _P, _I, _P, _P, _I, _I, _P, _P, _P, C.POINTER(HqScalars), _I, _P, _P, _P, _P]),
    "ddnm_hq_undo": (C.c_int, [_P, _P, _F, _F, _LL, _P]),
    "ddnm_data_transform": (C.c_int, [_P, _LL, _P, _P, _I, _I, _P, _P]),
    "ddnm_inverse_data_transform": (C.c_int, [_P, _LL, _I, _I, _P, _P]),
    "ddnm_finish_images": (C.c_int, [_P, _P, _I, _I, _I, _I, _I, _I, _P, _P, _P, _P]),
    "ddnm_conv_tc": (C.c_int, [_P, _I, _I, _I, _I, _P, _P, _I, _I, _I, _P, _I, _P, _P, _P, _P]),
    "ddnm_conv_direct": (C.c_int, [_P, _I, _I, _I, _I, _P, _P, _I, _I, _I, _P, _P]),
    "ddnm_conv_tc_bench": (C.c_int, [_I, _I, _I, _I, _I, _I, _I, C.POINTER(_F), C.POINTER(_D)]),
    "ddnm_gnconv_chunk_bench": (C.c_int, [_I, _I, _I, _I, _I, _I, _I, C.POINTER(_F)]),
    "ddnm_groupnorm": (C.c_int, [_P, _I, _I, _I, _I, _I, _P, _P, _F, _I, _P, _P]),
    "ddnm_conv_gn_tc": (C.c_int, [_P, _I, _I, _I, _I, _I, _P, _P, _F, _I, _P, _P, _I, _P, _I, _P, _P, _P, _I, C.POINTER(_F), _P]),
    "ddnm_tc_debug_gn_fused": (C.c_int, [_I]),
    "ddnm_tc_debug_force_bn": (C.c_int, [_I]),
    "ddnm_tc_debug_deal": (C.c_int, [_I]),
    "ddnm_tc_debug_pair_dual": (C.c_int, [_I]),
    "ddnm_tc_debug_dual_mode": (C.c_int, [_I]),
    "ddnm_tc_debug_pair_mode": (C.c_int, [_I]),
    "ddnm_tc_debug_halo": (C.c_int, [_I]),
    "ddnm_tc_debug_pingpong": (C.c_int, [_I]),
}
EXPORTS = ["ddnm_last_error"] + list(_SIGS)


def lib():
    """Load the library once; raise DDNMError if it is absent (no CPU / eager fallback exists)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise DDNMError(f"{LIB_PATH} not found: run `python -c 'import __graft_entry__ as g; g.build()'` first")
        L = C.CDLL(LIB_PATH)
        L.ddnm_last_error.restype = C.c_char_p
        L.ddnm_last_error.argtypes = []
        missing = [n for n in _SIGS if not hasattr(L, n)]
        if missing:
            raise DDNMError(f"{LIB_PATH} lacks symbols {missing}: stale build?")
        for name, (res, args) in _SIGS.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = res, args
        _lib = L
    return _lib


def check(rc):
    if rc != 0:
        raise DDNMError(lib().ddnm_last_error().decode("utf-8", "replace"))


def ptr(t):
    """Raw data pointer of a torch tensor (or None)."""
    return None if t is None else C.c_void_p(t.data_ptr())


def cur_stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)
