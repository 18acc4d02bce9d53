"""ctypes binding of csrc/libmapnet_b200.so (the C ABI in include/mapnet_b200.h).

Fails loudly: if the shared library is missing or a call returns non-zero a
RuntimeError carrying mapnet_last_error() is raised.  There is no CPU or
PyTorch fallback anywhere in this package.
"""
import ctypes
import os
from ctypes import c_char_p, c_float, c_int, c_int64, c_uint64, c_void_p, POINTER

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libmapnet_b200.so")

PREC = {"fp32": 0, "bf16": 1, "bf16_simt": 2, "tc_split": 3}
# precisions of the inference engine (mapnet_infer_*): fp8 exists there only, training stays in PREC
INFER_PREC = {"bf16": 1, "tc_split": 3, "fp8": 4}
N_F8_TENSORS = 33      # e4m3 activation tensors of the fp8 engine at ResNet-34: the pool output, 16 x (h, block output)
LOSS_MODE = {"posenet": 0, "mapnet": 1, "online": 2, "online_gps": 3}

_lib = None


class MapNetLibError(RuntimeError):
    pass


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise MapNetLibError(
            "geomapnet_b200: %s is missing -- build it with `python -m geomapnet_b200.build` "
            "(nvcc, sm_90a).  There is no fallback path." % LIB_PATH)
    L = ctypes.CDLL(LIB_PATH)
    L.mapnet_last_error.restype = c_char_p
    L.mapnet_abi_version.restype = c_int
    L.mapnet_trunk_create.argtypes = [POINTER(c_void_p), c_int, c_int, c_int, c_int, c_int]
    L.mapnet_trunk_destroy.argtypes = [c_void_p]
    L.mapnet_param_count.argtypes = [c_void_p]
    L.mapnet_param_info.argtypes = [c_void_p, c_int, c_char_p, c_int, POINTER(c_int), POINTER(c_int),
                                    POINTER(c_int64), POINTER(c_int64)]
    L.mapnet_param_layout.argtypes = [c_void_p, c_int]
    L.mapnet_param_layout.restype = c_int
    L.mapnet_params_numel.argtypes = [c_void_p]
    L.mapnet_params_numel.restype = c_int64
    L.mapnet_bufs_numel.argtypes = [c_void_p]
    L.mapnet_bufs_numel.restype = c_int64
    L.mapnet_forward.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_uint64,
                                 c_uint64, c_void_p, c_void_p]
    L.mapnet_backward.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p]
    L.mapnet_backward_part.argtypes = [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p]
    L.mapnet_backward_part.restype = c_int
    L.mapnet_grad_part_range.argtypes = [c_void_p, c_int, POINTER(c_int64), POINTER(c_int64)]
    L.mapnet_grad_part_range.restype = c_int
    L.mapnet_trunk_set_trainable.argtypes = [c_void_p, POINTER(ctypes.c_uint8), c_int]
    L.mapnet_trunk_set_trainable.restype = c_int
    L.mapnet_loss_fwd_bwd.argtypes = [c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p,
                                      c_void_p, c_void_p, c_void_p]
    L.mapnet_sqnorm.argtypes = [c_void_p, c_int64, c_void_p, c_void_p, c_void_p]
    L.mapnet_adam_step.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_float, c_float, c_float,
                                   c_float, c_float, c_int64, c_float, c_void_p, c_float, c_void_p]
    L.mapnet_adam_step_dev.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_float, c_float, c_float,
                                       c_float, c_float, c_void_p, c_float, c_void_p, c_float, c_void_p]
    L.mapnet_adam_step_dev.restype = c_int
    L.mapnet_sgd_step_dev.argtypes = [c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_float, ctypes.c_double,
                                      c_float, c_int, c_void_p, c_float, c_void_p, c_float, c_void_p]
    L.mapnet_sgd_step_dev.restype = c_int
    L.mapnet_rmsprop_step_dev.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_void_p,
                                          ctypes.c_double, c_float, c_float, c_float, c_void_p, c_float, c_void_p,
                                          c_float, c_void_p]
    L.mapnet_rmsprop_step_dev.restype = c_int
    L.mapnet_test_conv.argtypes = [c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p,
                                   c_void_p, c_void_p, c_void_p, c_void_p]
    L.mapnet_test_conv_ex.argtypes = [c_int] * 9 + [c_void_p] * 4 + [c_float, c_void_p, c_void_p]
    L.mapnet_test_conv_ex.restype = c_int
    L.mapnet_test_stem.argtypes = [c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]
    L.mapnet_test_stem.restype = c_int
    L.mapnet_test_dgrad_shortcut.argtypes = [c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                             c_void_p, c_void_p]
    L.mapnet_test_dgrad_shortcut.restype = c_int
    L.mapnet_preprocess_create.argtypes = [POINTER(c_void_p), c_int, c_int, c_int, c_int]
    L.mapnet_preprocess_output_size.argtypes = [c_void_p, POINTER(c_int), POINTER(c_int)]
    L.mapnet_preprocess_run.argtypes = [c_void_p, c_void_p, c_int, POINTER(c_float), POINTER(c_float), c_void_p, c_void_p,
                                        c_void_p]
    L.mapnet_preprocess_destroy.argtypes = [c_void_p]
    L.mapnet_preprocess_run_ex.argtypes = [c_void_p, c_void_p, c_int, c_void_p, c_void_p, POINTER(c_float), POINTER(c_float),
                                           c_void_p, c_void_p, c_void_p]
    for name in ("mapnet_preprocess_create", "mapnet_preprocess_output_size", "mapnet_preprocess_run",
                 "mapnet_preprocess_run_ex", "mapnet_preprocess_destroy"):
        getattr(L, name).restype = c_int
    L.mapnet_frame_cache_create.argtypes = [POINTER(c_void_p), c_int, c_int, c_int, c_int, c_int, c_int, c_int]
    L.mapnet_frame_cache_ingest.argtypes = [c_void_p, c_void_p, c_int, c_int, c_void_p]
    L.mapnet_frame_cache_assemble.argtypes = [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int,
                                              POINTER(c_float), POINTER(c_float), c_void_p, c_void_p, c_void_p]
    L.mapnet_frame_cache_destroy.argtypes = [c_void_p]
    for name in ("mapnet_frame_cache_create", "mapnet_frame_cache_ingest", "mapnet_frame_cache_assemble",
                 "mapnet_frame_cache_destroy"):
        getattr(L, name).restype = c_int
    L.mapnet_eval_windows.argtypes = [c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int,
                                      c_void_p, c_void_p, c_void_p, c_void_p]
    L.mapnet_eval_windows.restype = c_int
    L.mapnet_batch_losses.argtypes = [c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int,
                                      c_void_p, c_void_p, c_void_p]
    L.mapnet_batch_losses.restype = c_int
    L.mapnet_pose_post.argtypes =[c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p]
    L.mapnet_pose_post.restype = c_int
    L.mapnet_pgo_optimize.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, ctypes.c_double, ctypes.c_double,
                                      ctypes.c_double, ctypes.c_double, c_int, c_int, c_void_p, c_void_p]
    L.mapnet_pgo_optimize.restype = c_int
    L.mapnet_test_conv_epilogue.argtypes = [c_int] * 8 + [c_void_p] * 10 + [c_void_p]
    L.mapnet_test_conv_epilogue.restype = c_int
    L.mapnet_test_plan_describe.argtypes = [c_int] * 9 + [c_char_p, c_int]
    L.mapnet_test_plan_describe.restype = c_int
    L.mapnet_launch_count.restype = ctypes.c_ulonglong
    L.mapnet_profile.argtypes = [c_void_p, c_int]
    L.mapnet_profile.restype = c_int
    L.mapnet_profile_read.argtypes = [c_void_p, POINTER(ctypes.c_double), POINTER(ctypes.c_double), POINTER(c_int)]
    L.mapnet_profile_read.restype = c_int
    L.mapnet_bench_conv.argtypes = [c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                    c_void_p, c_void_p, c_int, POINTER(c_float)]
    L.mapnet_bench_conv.restype = c_int
    L.mapnet_test_conv_affine.argtypes = [c_int] * 8 + [c_void_p] * 5 + [c_int, c_void_p, c_void_p]
    L.mapnet_test_conv_affine.restype = c_int
    L.mapnet_infer_create.argtypes = [POINTER(c_void_p), c_int, c_int, c_int, c_int, c_int]
    L.mapnet_infer_load.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p]
    L.mapnet_infer_forward.argtypes = [c_void_p, c_void_p, c_int, c_float, c_uint64, c_uint64, c_void_p, c_void_p]
    L.mapnet_infer_arena_bytes.argtypes = [c_int, c_int, c_int, c_int]
    L.mapnet_infer_arena_bytes.restype = c_int64
    L.mapnet_infer_destroy.argtypes = [c_void_p]
    L.mapnet_infer_calibrate.argtypes = [c_void_p, c_void_p, c_int, c_void_p]
    L.mapnet_infer_act_scales.argtypes = [c_void_p, POINTER(c_float), c_int]
    L.mapnet_test_conv_fp8.argtypes = [c_int] * 7 + [c_void_p] * 7 + [c_int, c_void_p, c_void_p, c_void_p]
    L.mapnet_test_conv_fp8.restype = c_int
    L.mapnet_test_bn_forward.argtypes = [c_int] * 4 + [c_int64, c_int] + [c_void_p] * 5 + [c_int, c_void_p, c_void_p]
    L.mapnet_test_bn_backward.argtypes = [c_int] * 3 + [c_int64, c_int] + [c_void_p] * 9 + [c_int, c_float, c_void_p,
                                                                                              c_void_p]
    L.mapnet_test_stem_pool.argtypes = [c_int] * 6 + [c_void_p] * 8 + [c_int, c_void_p, c_void_p]
    L.mapnet_test_gap.argtypes = [c_int] * 4 + [c_void_p] * 5
    for name in ("mapnet_test_bn_forward", "mapnet_test_bn_backward", "mapnet_test_stem_pool", "mapnet_test_gap"):
        getattr(L, name).restype = c_int
    for name in ("mapnet_infer_create", "mapnet_infer_load", "mapnet_infer_forward", "mapnet_infer_destroy",
                 "mapnet_infer_calibrate", "mapnet_infer_act_scales"):
        getattr(L, name).restype = c_int
    for name in ("mapnet_trunk_create", "mapnet_trunk_destroy", "mapnet_param_count", "mapnet_param_info",
                 "mapnet_forward", "mapnet_backward", "mapnet_loss_fwd_bwd", "mapnet_sqnorm",
                 "mapnet_adam_step", "mapnet_test_conv"):
        getattr(L, name).restype = c_int
    _lib = L
    return L


EXPORTED = ["mapnet_last_error", "mapnet_abi_version", "mapnet_trunk_create", "mapnet_trunk_destroy",
            "mapnet_param_count", "mapnet_param_info", "mapnet_param_layout", "mapnet_params_numel", "mapnet_bufs_numel",
            "mapnet_forward", "mapnet_backward", "mapnet_loss_fwd_bwd", "mapnet_sqnorm", "mapnet_adam_step",
            "mapnet_test_conv", "mapnet_launch_count", "mapnet_profile", "mapnet_profile_read",
            "mapnet_adam_step_dev", "mapnet_bench_conv", "mapnet_test_stem",
            "mapnet_test_dgrad_shortcut", "mapnet_test_plan_describe", "mapnet_preprocess_create",
            "mapnet_preprocess_output_size", "mapnet_preprocess_run", "mapnet_preprocess_destroy",
            "mapnet_backward_part", "mapnet_grad_part_range", "mapnet_preprocess_run_ex", "mapnet_test_conv_epilogue", "mapnet_pose_post", "mapnet_pgo_optimize",
            "mapnet_sgd_step_dev", "mapnet_rmsprop_step_dev", "mapnet_test_conv_affine", "mapnet_infer_create",
            "mapnet_infer_load", "mapnet_infer_forward", "mapnet_infer_arena_bytes", "mapnet_infer_destroy",
            "mapnet_frame_cache_create", "mapnet_frame_cache_ingest", "mapnet_frame_cache_assemble",
            "mapnet_frame_cache_destroy", "mapnet_infer_calibrate", "mapnet_infer_act_scales", "mapnet_test_conv_fp8",
            "mapnet_test_bn_forward", "mapnet_test_bn_backward", "mapnet_test_stem_pool", "mapnet_test_gap",
            "mapnet_trunk_set_trainable", "mapnet_test_conv_ex", "mapnet_eval_windows",
            "mapnet_batch_losses"]
UINT64_MAX = 0xFFFFFFFFFFFFFFFF


def check(rc, what):
    if rc != 0:
        msg = lib().mapnet_last_error()
        raise MapNetLibError("%s failed (rc=%d): %s" % (what, rc, msg.decode() if msg else "?"))


def stream_ptr():
    import torch
    return c_void_p(torch.cuda.current_stream().cuda_stream)


class Trunk(object):
    """Owns one mapnet_trunk_t handle."""

    def __init__(self, max_B, H, W, feat_dim, precision):
        self.h = c_void_p()
        self.max_B, self.H, self.W, self.feat_dim, self.precision = max_B, H, W, feat_dim, precision
        self.trainable = None         # the mask last passed to mapnet_trunk_set_trainable
        check(lib().mapnet_trunk_create(ctypes.byref(self.h), max_B, H, W, feat_dim, PREC[precision]),
              "mapnet_trunk_create")

    def set_trainable(self, mask):
        """mask: one flag per trainable entry (kind 0) of the parameter table, in table order.  The handle is told only
        when the mask differs from the one last passed."""
        mask = tuple(bool(m) for m in mask)
        if mask == self.trainable:
            return
        buf = (ctypes.c_uint8 * len(mask))(*mask)
        check(lib().mapnet_trunk_set_trainable(self.h, buf, len(mask)), "mapnet_trunk_set_trainable")
        self.trainable = mask

    def table(self):
        L = lib()
        n = L.mapnet_param_count(self.h)
        out = []
        name = ctypes.create_string_buffer(128)
        kind, ndim, off = c_int(), c_int(), c_int64()
        shape = (c_int64 * 4)()
        for i in range(n):
            check(L.mapnet_param_info(self.h, i, name, 128, ctypes.byref(kind), ctypes.byref(ndim), shape,
                                      ctypes.byref(off)), "mapnet_param_info")
            out.append((name.value.decode(), kind.value, tuple(shape[k] for k in range(ndim.value)), off.value))
        return out, L.mapnet_params_numel(self.h), L.mapnet_bufs_numel(self.h)

    def layouts(self):
        """{entry name: 1} for the conv weights the flat buffers hold in [Co][KH][KW][Ci] order (mapnet_param_layout)."""
        L = lib()
        names = [e[0] for e in self.table()[0]]
        return {nm: 1 for i, nm in enumerate(names) if L.mapnet_param_layout(self.h, i) == 1}

    def grad_part_ranges(self):
        """[(lo, hi)] float ranges of the flat gradient buffer completed by backward parts 0, 1, 2."""
        out = []
        lo, hi = c_int64(), c_int64()
        for part in range(3):
            check(lib().mapnet_grad_part_range(self.h, part, ctypes.byref(lo), ctypes.byref(hi)), "mapnet_grad_part_range")
            out.append((lo.value, hi.value))
        return out

    def close(self):
        if self.h:
            lib().mapnet_trunk_destroy(self.h)
            self.h = c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Infer(object):
    """Owns one mapnet_infer_t handle (the eval-mode inference engine of one (max_B, H, W))."""

    def __init__(self, max_B, H, W, feat_dim, precision):
        self.h = c_void_p()
        self.max_B, self.H, self.W, self.feat_dim, self.precision = max_B, H, W, feat_dim, precision
        check(lib().mapnet_infer_create(ctypes.byref(self.h), max_B, H, W, feat_dim,
                                        INFER_PREC.get(precision, PREC.get(precision, -1))), "mapnet_infer_create")

    def load(self, params_flat, bufs_flat):
        check(lib().mapnet_infer_load(self.h, params_flat.data_ptr(), bufs_flat.data_ptr(), stream_ptr()),
              "mapnet_infer_load")

    def calibrate(self, x):
        """fp8 engines: activation scales from frames x [B,3,H,W] (float32, contiguous, on the device)"""
        check(lib().mapnet_infer_calibrate(self.h, x.data_ptr(), x.shape[0], stream_ptr()), "mapnet_infer_calibrate")

    def act_scales(self):
        """fp8 engines: the activation scales in schedule order (pool output, then each block's h and output)"""
        import torch
        torch.cuda.current_stream().synchronize()      # the scales of a calibration queued on this stream
        buf = (c_float * N_F8_TENSORS)()
        check(lib().mapnet_infer_act_scales(self.h, buf, N_F8_TENSORS), "mapnet_infer_act_scales")
        return list(buf)

    def forward(self, x, pred, droprate, seed, step=UINT64_MAX):
        check(lib().mapnet_infer_forward(self.h, x.data_ptr(), x.shape[0], float(droprate), int(seed), int(step),
                                         pred.data_ptr(), stream_ptr()), "mapnet_infer_forward")

    def close(self):
        if self.h:
            lib().mapnet_infer_destroy(self.h)
            self.h = c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
