"""ctypes binding of libpmvs_b200.so (the C ABI declared in include/pmvs_b200.h).

The library is the product: there is no CPU or PyTorch fallback.  Importing this module
fails loudly if the shared object has not been built (``python -c "import __graft_entry__
as g; g.build()"`` or ``pointmvsnet_b200/csrc/build.sh``).
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libpmvs_b200.so")

if not os.path.exists(LIB_PATH):
    raise ImportError(
        "pointmvsnet_b200: %s is missing -- build it with pointmvsnet_b200/csrc/build.sh "
        "(nvcc, sm_90a).  There is no CPU fallback." % LIB_PATH)

lib = C.CDLL(LIB_PATH)

c_float_p = C.c_void_p
c_stream = C.c_void_p


class FlowWeights(C.Structure):
    _fields_ = [
        ("ec_w12", C.c_void_p * 3), ("ec_gamma", C.c_void_p * 3), ("ec_beta", C.c_void_p * 3),
        ("mlp_w", C.c_void_p * 4), ("mlp_gamma", C.c_void_p * 3), ("mlp_beta", C.c_void_p * 3),
        ("ec_run_mean", C.c_void_p * 3), ("ec_run_var", C.c_void_p * 3),
        ("mlp_run_mean", C.c_void_p * 3), ("mlp_run_var", C.c_void_p * 3),
        ("momentum", C.c_float), ("eps", C.c_float),
        ("ec_nbt", C.c_void_p * 3), ("mlp_nbt", C.c_void_p * 3),
    ]


class FlowShape(C.Structure):
    _fields_ = [
        ("B", C.c_int), ("V", C.c_int), ("pyr_h", C.c_int * 3), ("pyr_w", C.c_int * 3),
        ("prev_h", C.c_int), ("prev_w", C.c_int), ("flow_h", C.c_int), ("flow_w", C.c_int),
        ("image_scale", C.c_float), ("ratio", C.c_int), ("is_test", C.c_int), ("interval_scale", C.c_float),
        ("sub_begin", C.c_int), ("sub_count", C.c_int), ("bn_eval", C.c_int),
    ]


class FlowGrads(C.Structure):
    _fields_ = [
        ("ec_dw12", C.c_void_p * 3), ("ec_dgamma", C.c_void_p * 3), ("ec_dbeta", C.c_void_p * 3),
        ("mlp_dw", C.c_void_p * 4), ("mlp_dgamma", C.c_void_p * 3), ("mlp_dbeta", C.c_void_p * 3),
        ("dpyramids_cl", C.c_void_p * 3), ("ddepth_prev", C.c_void_p),
    ]


class ConvBnWeights(C.Structure):
    """pmvs_conv_bn_weights (pmvs_volume_weights, pmvs_image_weights)"""
    _fields_ = [
        ("weight", C.c_void_p * 11), ("gamma", C.c_void_p * 10), ("beta", C.c_void_p * 10),
        ("running_mean", C.c_void_p * 10), ("running_var", C.c_void_p * 10), ("eps", C.c_float * 10),
    ]


class ConvBnGrads(C.Structure):
    """pmvs_conv_bn_grads (pmvs_volume_grads, pmvs_image_grads)"""
    _fields_ = [("weight", C.c_void_p * 11), ("gamma", C.c_void_p * 10), ("beta", C.c_void_p * 10)]


# the per-tower names, kept for existing callers as the C header keeps its typedefs
VolumeWeights = ImageWeights = ConvBnWeights
VolumeGrads = ImageGrads = ConvBnGrads


class DepthTerms(C.Structure):
    _fields_ = [("pred", C.c_void_p * 3), ("h", C.c_int * 3), ("w", C.c_int * 3), ("T", C.c_int)]


def _sig(name, restype, argtypes):
    fn = getattr(lib, name)
    fn.restype = restype
    fn.argtypes = argtypes
    return fn


P, I, LL, F = C.c_void_p, C.c_int, C.c_longlong, C.c_float
_sig("pmvs_version", I, [])
_sig("pmvs_last_error", C.c_char_p, [])
_sig("pmvs_launch_count", C.c_ulonglong, [])
_sig("pmvs_set_gemm_mode", I, [I])
_sig("pmvs_get_gemm_mode", I, [])
_sig("pmvs_set_option", I, [I, I])
_sig("pmvs_get_option", I, [I])
_sig("pmvs_profile_enable", I, [I])
_sig("pmvs_profile_collect", I, [C.c_char_p, C.c_size_t, P, I])
_sig("pmvs_gather_knn_forward", I, [P, P, P, I, I, I, I, P])
_sig("pmvs_gather_knn_backward", I, [P, P, P, I, I, I, I, P])
_sig("pmvs_gather_knn_backward_det_workspace_bytes", C.c_size_t, [I, I, I])
_sig("pmvs_gather_knn_backward_det", I, [P, P, P, I, I, I, I, P, C.c_size_t, P])
_sig("pmvs_knn3d", I, [P, P, P, I, I, I, I, I, I, P])
_sig("pmvs_feature_fetch", I, [P, P, P, P, P, I, I, I, I, I, I, P])
_sig("pmvs_feature_fetch_backward", I, [P, P, P, P, P, I, I, I, I, I, I, P])
_sig("pmvs_feature_fetch_backward_det_workspace_bytes", C.c_size_t, [I, I, I, I, I, I])
_sig("pmvs_feature_fetch_backward_det", I, [P, P, P, P, P, I, I, I, I, I, I, P, C.c_size_t, P])
_sig("pmvs_feature_fetch_taps", I, [P, P, P, P, P, I, I, I, I, I, P])
_sig("pmvs_cost_volume", I, [P, P, P, P, C.c_size_t, I, I, I, I, I, I, I, P])
_sig("pmvs_cost_volume_backward_workspace_bytes", C.c_size_t, [I, I, I, I, I, I])
_sig("pmvs_cost_volume_backward", I, [P, P, P, P, P, C.c_size_t, I, I, I, I, I, I, I, P])
_sig("pmvs_fuse_depth_maps_workspace_bytes", C.c_size_t, [I, I, I])
_sig("pmvs_fuse_depth_maps", I, [P, P, I, I, I, I, F, F, P, P, P, P, C.c_size_t, P])
_sig("pmvs_thin_cloud_workspace_bytes", C.c_size_t, [I])
_sig("pmvs_thin_cloud", I, [P, P, I, F, F, I, I, P, P, P, C.c_size_t, P])
_sig("pmvs_nearest_distances_workspace_bytes", C.c_size_t, [I])
_sig("pmvs_nearest_distances", I, [P, I, P, I, F, F, P, P, C.c_size_t, P])
_sig("pmvs_cloud_filter", I, [P, I, P, F, P, P, F, P, P, P])
_sig("pmvs_volume_conv_workspace_bytes", C.c_size_t, [I, I, I, I, I, I])
_sig("pmvs_volume_conv", I, [P, C.POINTER(ConvBnWeights), I, P, P, P, C.c_size_t, I, I, I, I, I, I, P])
_sig("pmvs_coarse_depth", I, [P, P, I, I, I, I, I, P, P, P])
_sig("pmvs_volume_conv_backward_workspace_bytes", C.c_size_t, [I, I, I, I, I, I])
_sig("pmvs_volume_conv_backward", I, [P, C.POINTER(ConvBnWeights), I, P, P, P, P, C.POINTER(ConvBnGrads), P,
                                      C.c_size_t, I, I, I, I, I, I, P])
_sig("pmvs_coarse_depth_backward", I, [P, P, P, P, I, I, I, I, I, P])
_sig("pmvs_image_conv_workspace_bytes", C.c_size_t, [I, I, I, I, I])
_sig("pmvs_image_conv", I, [P, C.POINTER(ConvBnWeights), I, C.POINTER(C.c_void_p * 4), I, P, P, C.c_size_t, I, I, I,
                            I, I, P])
_sig("pmvs_image_conv_keep_workspace_bytes", C.c_size_t, [I, I, I, I, I])
_sig("pmvs_image_conv_keep", I, [P, C.POINTER(ConvBnWeights), I, C.POINTER(C.c_void_p * 4), I, P, P, C.c_size_t, I,
                                 I, I, I, I, P])
_sig("pmvs_image_conv_backward_workspace_bytes", C.c_size_t, [I, I, I, I, I])
_sig("pmvs_image_conv_backward", I, [P, C.POINTER(ConvBnWeights), I, P, P, C.POINTER(C.c_void_p * 4), I,
                                     C.POINTER(ConvBnGrads), P, C.c_size_t, I, I, I, I, I, P])
_sig("pmvs_transpose", I, [P, P, I, I, I, P])
_sig("pmvs_idx64_to_idx32", I, [P, P, LL, P])
_sig("pmvs_edgeconv_pm", I, [P, I, P, P, P, P, F, I, I, P, I, P, P, I, I, I, I, I, I, P])
_sig("pmvs_edgeconv_pm_backward_workspace_bytes", C.c_size_t, [I, I, I, I, I])
_sig("pmvs_edgeconv_pm_backward", I, [P, I, P, P, P, P, P, F, I, I, P, P, P, I, P, I, P, P, P, P, C.c_size_t,
                                      I, I, I, I, I, P])
_sig("pmvs_linear_pm", I, [P, I, P, P, I, I, I, I, I, P, P, P, C.c_double, F, P, P])
_sig("pmvs_point_flow_workspace_bytes", C.c_size_t, [C.POINTER(FlowShape)])
_sig("pmvs_point_flow_iter", I, [C.POINTER(FlowShape), C.POINTER(FlowWeights), C.POINTER(C.c_void_p * 3),
                                 P, P, P, P, P, P, P, P, C.c_size_t, P])
_sig("pmvs_pyramid_to_channels_last", I, [P, P, I, I, I, I, P])
_sig("pmvs_point_flow_debug_offsets", I, [C.POINTER(FlowShape), C.POINTER(C.c_size_t * 10)])
_sig("pmvs_point_flow_debug_feature", I, [C.POINTER(FlowShape), P, P, P])
_sig("pmvs_point_flow_backward_workspace_bytes", C.c_size_t, [C.POINTER(FlowShape)])
_sig("pmvs_point_flow_backward", I, [C.POINTER(FlowShape), C.POINTER(FlowWeights), C.POINTER(C.c_void_p * 3),
                                     P, P, P, P, P, P, P, P, C.POINTER(FlowGrads), P, C.c_size_t, P])
_sig("pmvs_point_flow_eval_keep_workspace_bytes", C.c_size_t, [C.POINTER(FlowShape)])
_sig("pmvs_point_flow_eval_keep", I, [C.POINTER(FlowShape), C.POINTER(FlowWeights), C.POINTER(C.c_void_p * 3),
                                      P, P, P, P, P, P, P, P, C.c_size_t, P])
_sig("pmvs_point_flow_eval_backward_workspace_bytes", C.c_size_t, [C.POINTER(FlowShape)])
_sig("pmvs_point_flow_eval_backward", I, [C.POINTER(FlowShape), C.POINTER(FlowWeights), C.POINTER(C.c_void_p * 3),
                                          P, P, P, P, P, P, P, P, C.POINTER(FlowGrads), P, C.c_size_t, P])
_sig("pmvs_point_flow_backward_debug_offsets", I, [C.POINTER(FlowShape), I, C.POINTER(C.c_size_t * 7)])
_sig("pmvs_depth_loss", I, [C.POINTER(DepthTerms), P, I, I, P, I, I, F, P, P, P, P])
_sig("pmvs_depth_loss_backward", I, [C.POINTER(DepthTerms), P, I, I, P, I, I, P, P, C.POINTER(C.c_void_p * 3), P])
_sig("pmvs_prepare_views_workspace_bytes", C.c_size_t, [I, I, I, I, C.c_double, I, I, I, I])
_sig("pmvs_prepare_views", I, [P, I, I, I, I, C.c_double, I, I, I, I, P, P, P, C.c_size_t, P])
_sig("pmvs_probability_filter_workspace_bytes", C.c_size_t, [I, I, I, I, I, I, I, I])
_sig("pmvs_probability_filter", I, [P, P, P, I, I, I, I, I, I, I, F, F, I, P, C.c_size_t, P, P, C.c_size_t, P])

EXPORTED = [
    "pmvs_version", "pmvs_last_error", "pmvs_launch_count", "pmvs_set_option", "pmvs_get_option", "pmvs_profile_enable", "pmvs_profile_collect", "pmvs_set_gemm_mode", "pmvs_get_gemm_mode", "pmvs_gather_knn_forward",
    "pmvs_gather_knn_backward", "pmvs_gather_knn_backward_det_workspace_bytes", "pmvs_gather_knn_backward_det", "pmvs_knn3d", "pmvs_feature_fetch", "pmvs_feature_fetch_backward",
    "pmvs_feature_fetch_backward_det_workspace_bytes", "pmvs_feature_fetch_backward_det", "pmvs_feature_fetch_taps",
    "pmvs_cost_volume", "pmvs_cost_volume_backward_workspace_bytes", "pmvs_cost_volume_backward",
    "pmvs_fuse_depth_maps_workspace_bytes", "pmvs_fuse_depth_maps", "pmvs_thin_cloud_workspace_bytes",
    "pmvs_thin_cloud", "pmvs_nearest_distances_workspace_bytes", "pmvs_nearest_distances", "pmvs_cloud_filter",
    "pmvs_volume_conv_workspace_bytes", "pmvs_volume_conv", "pmvs_coarse_depth",
    "pmvs_volume_conv_backward_workspace_bytes", "pmvs_volume_conv_backward", "pmvs_coarse_depth_backward",
    "pmvs_image_conv_workspace_bytes", "pmvs_image_conv", "pmvs_image_conv_keep_workspace_bytes",
    "pmvs_image_conv_keep", "pmvs_image_conv_backward_workspace_bytes", "pmvs_image_conv_backward",
    "pmvs_transpose", "pmvs_idx64_to_idx32", "pmvs_edgeconv_pm", "pmvs_edgeconv_pm_backward_workspace_bytes", "pmvs_edgeconv_pm_backward", "pmvs_linear_pm", "pmvs_point_flow_workspace_bytes",
    "pmvs_point_flow_iter", "pmvs_pyramid_to_channels_last", "pmvs_point_flow_debug_offsets",
    "pmvs_point_flow_debug_feature", "pmvs_point_flow_backward_workspace_bytes", "pmvs_point_flow_backward",
    "pmvs_depth_loss", "pmvs_depth_loss_backward", "pmvs_point_flow_eval_keep_workspace_bytes",
    "pmvs_point_flow_eval_keep", "pmvs_point_flow_eval_backward_workspace_bytes", "pmvs_point_flow_eval_backward",
    "pmvs_point_flow_backward_debug_offsets", "pmvs_prepare_views_workspace_bytes", "pmvs_prepare_views",
    "pmvs_probability_filter_workspace_bytes", "pmvs_probability_filter",
]


def check(rc):
    """Error convention of the reference extension: c10 error -> RuntimeError
    (functions/csrc/gather_knn_kernel.cu:10-12)."""
    if rc != 0:
        raise RuntimeError("libpmvs_b200: " + lib.pmvs_last_error().decode("utf-8", "replace"))


def stream_ptr():
    return torch.cuda.current_stream().cuda_stream


def ptr(t):
    return None if t is None else t.data_ptr()


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError("pointmvsnet_b200 operators need CUDA tensors (sm_90a); there is no CPU fallback")


def f32c(t):
    """contiguous fp32 view/copy"""
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


def workspace(nbytes, device):
    """a device workspace of `nbytes` bytes, a library size function's result (0: the library's error is raised).
    The caching allocator aligns blocks to 512 bytes, more than the 256 the library needs."""
    if nbytes == 0:
        check(1)
    return torch.empty(nbytes, device=device, dtype=torch.uint8)


def launch_count():
    return int(lib.pmvs_launch_count())


def profile_enable(on):
    lib.pmvs_profile_enable(1 if on else 0)


def profile_collect(max_records=65536):
    """-> list of (kernel name, milliseconds) in launch order"""
    names = C.create_string_buffer(max_records * 24)
    ms = (C.c_float * max_records)()
    n = lib.pmvs_profile_collect(names, len(names), C.cast(ms, C.c_void_p), max_records)
    nm = names.value.decode().split("\n")[:n]
    return [(nm[i], float(ms[i])) for i in range(n)]


def set_gemm_mode(mode):
    """0: fp32 SIMT, 1: TF32 tensor cores, 3: 3xTF32 tensor cores (default)"""
    check(lib.pmvs_set_gemm_mode(int(mode)))


# implementation switches (include/pmvs_b200.h PMVS_OPT_*): which kernel family serves a stage of the fused path
OPTIONS = {"edge": 1, "knn": 2, "fetch": 3, "gemm": 4, "debug_idx": 5, "gemm_strict": 6}


def set_option(name, value):
    check(lib.pmvs_set_option(OPTIONS[name], int(value)))


def get_option(name):
    return int(lib.pmvs_get_option(OPTIONS[name]))


def _options_from_env():
    """PMVS_OPTIONS="edge=0,knn=0" selects the older kernel families (A/B measurements, bisecting)."""
    spec = os.environ.get("PMVS_OPTIONS", "")
    for item in spec.split(","):
        if "=" in item:
            k, v = item.split("=", 1)
            set_option(k.strip(), int(v))


_options_from_env()
