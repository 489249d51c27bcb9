"""ctypes binding of the C-ABI in include/ltr_b200.h (libltr_b200.so).

This is the stub a Python maintainer would add on the reference side; it contains no arithmetic.  The
library is CUDA-only: loading fails loudly when it has not been built, and `Context()` raises when
no sm_90 device is usable -- there is no CPU fallback.
"""
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libltr_b200.so")
_LIB = None

MODE_HD, MODE_ND, MODE_PD = 0, 1, 2
SCANSIDE_MAP, SCANSIDE_SCAN_MINUS_MAP = 0, 1   # ltr_scanside_criterion
ICP_ITERATIONS, ICP_TRANSFORM, ICP_ABS_MSE, ICP_REL_MSE, ICP_NO_CORRESPONDENCES = 1, 2, 3, 4, 5   # ltr_icp_exit
LTR_OK = 0


class LtrError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"ltr error {code}: {msg}")
        self.code = code


class Config(ctypes.Structure):
    _fields_ = [("device", ctypes.c_int32), ("vfov_deg", ctypes.c_float), ("hfov_deg", ctypes.c_float),
                ("lidar2base", ctypes.c_double * 16), ("base2lidar", ctypes.c_double * 16),
                ("transform_order", ctypes.c_int32), ("keyframe_batch", ctypes.c_int32), ("fast_path", ctypes.c_int32)]


class IcpParams(ctypes.Structure):
    _fields_ = [("max_correspondence_distance", ctypes.c_double), ("max_iterations", ctypes.c_int32),
                ("transformation_epsilon", ctypes.c_double), ("euclidean_fitness_epsilon", ctypes.c_double),
                ("mse_threshold_absolute", ctypes.c_double), ("min_correspondences", ctypes.c_int32), ("source_leaf", ctypes.c_float)]


EXPORTS = [
    "ltr_config_default", "ltr_create", "ltr_destroy", "ltr_last_error", "ltr_synchronize", "ltr_kernel_launches", "ltr_voxel_shortcuts", "ltr_memory_stats",
    "ltr_cloud_upload", "ltr_cloud_size", "ltr_cloud_download", "ltr_cloud_free", "ltr_cloud_copy", "ltr_cloud_concat", "ltr_cloud_slice",
    "ltr_cloud_device_ptrs", "ltr_cloud_alloc", "ltr_scanset_upload", "ltr_scanset_info", "ltr_scanset_download",
    "ltr_scanset_free", "ltr_scanset_concat_per_keyframe", "ltr_scanset_flatten", "ltr_poses_upload", "ltr_poses_free",
    "ltr_preclean", "ltr_merge_scans_global", "ltr_voxel_centroid", "ltr_voxel_centroid_per_keyframe", "ltr_voxel_grid", "ltr_voxel_grid_per_keyframe", "ltr_remove_pass", "ltr_remove_pass_adaptive", "ltr_remove_pass_ball", "ltr_scan_images_release",
    "ltr_flags_device_ptr", "ltr_flags_download", "ltr_flags_upload", "ltr_apply_partition", "ltr_parse_projected",
    "ltr_knn_diff", "ltr_knn_split_cloud", "ltr_knn_split_per_keyframe", "ltr_scanside_split", "ltr_scanside_stats", "ltr_icp_params_default", "ltr_icp_refine", "ltr_knn_diff_refined", "ltr_icp_refine_scanside", "ltr_scanside_split_refined", "ltr_debug_pixel_index", "ltr_debug_scan_rimg", "ltr_debug_exact_knn_avg", "ltr_debug_nearest", "ltr_debug_fast_project", "ltr_debug_atan_sweep", "ltr_debug_margins", "ltr_debug_voxel_distributed", "ltr_reset_rimg_size", "ltr_last_pass_stats", "ltr_profile_get", "ltr_profile_reset", "ltr_timer_start", "ltr_timer_stop", "ltr_trace_dump",
    "ltr_pinned_alloc", "ltr_pinned_free", "ltr_nccl_unique_id", "ltr_nccl_init", "ltr_nccl_split", "ltr_nccl_info", "ltr_nccl_destroy", "ltr_nccl_version", "ltr_nccl_allreduce_flags",
    "ltr_nccl_allgather_clouds", "ltr_nccl_exchange_clouds", "ltr_nccl_voxel_centroid_merged", "ltr_nccl_allgather_i64", "ltr_nccl_max_f64", "ltr_nccl_barrier", "ltr_stream_handle",
]


def lib():
    """Loads libltr_b200.so (built by `make -C lt_mapper_b200/csrc` / __graft_entry__.build())."""
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'`; "
                          "lt_mapper_b200 has no CPU fallback")
    L = ctypes.CDLL(LIB_PATH)
    vp, i32, i64, f32 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_float
    P = ctypes.POINTER
    L.ltr_config_default.argtypes = [P(Config)]
    L.ltr_config_default.restype = None
    L.ltr_create.argtypes = [P(vp), P(Config)]
    L.ltr_destroy.argtypes = [vp]
    L.ltr_destroy.restype = None
    L.ltr_last_error.argtypes = [vp]
    L.ltr_last_error.restype = ctypes.c_char_p
    L.ltr_synchronize.argtypes = [vp]
    L.ltr_kernel_launches.argtypes = [vp]
    L.ltr_kernel_launches.restype = i64
    L.ltr_voxel_shortcuts.argtypes = [vp]
    L.ltr_voxel_shortcuts.restype = i64
    L.ltr_memory_stats.argtypes = [vp, vp]
    L.ltr_cloud_upload.argtypes = [vp, vp, i64, P(i32)]
    L.ltr_cloud_alloc.argtypes = [vp, i64, P(i32)]
    L.ltr_cloud_size.argtypes = [vp, i32, P(i64)]
    L.ltr_cloud_download.argtypes = [vp, i32, vp, i64, P(i64)]
    L.ltr_cloud_free.argtypes = [vp, i32]
    L.ltr_cloud_copy.argtypes = [vp, i32, P(i32)]
    L.ltr_cloud_concat.argtypes = [vp, i32, i32, P(i32)]
    L.ltr_cloud_slice.argtypes = [vp, i32, i64, i64, P(i32)]
    L.ltr_cloud_device_ptrs.argtypes = [vp, i32, P(vp), P(vp), P(vp), P(vp), P(i64)]
    L.ltr_scanset_upload.argtypes = [vp, vp, vp, i32, P(i32)]
    L.ltr_scanset_info.argtypes = [vp, i32, P(i32), P(i64)]
    L.ltr_scanset_download.argtypes = [vp, i32, vp, i64, vp]
    L.ltr_scanset_free.argtypes = [vp, i32]
    L.ltr_scanset_concat_per_keyframe.argtypes = [vp, i32, i32, P(i32)]
    L.ltr_scanset_flatten.argtypes = [vp, i32, P(i32)]
    L.ltr_poses_upload.argtypes = [vp, vp, vp, i32, P(i32)]
    L.ltr_poses_free.argtypes = [vp, i32]
    L.ltr_preclean.argtypes = [vp, i32, f32, P(i32)]
    L.ltr_merge_scans_global.argtypes = [vp, i32, i32, P(i32)]
    L.ltr_voxel_centroid.argtypes = [vp, i32, f32, P(i32)]
    L.ltr_voxel_centroid_per_keyframe.argtypes = [vp, i32, f32, P(i32)]
    L.ltr_voxel_grid.argtypes = [vp, i32, f32, P(i32), P(i32)]
    L.ltr_voxel_grid_per_keyframe.argtypes = [vp, i32, f32, P(i32), P(i32)]
    L.ltr_remove_pass.argtypes = [vp, i32, i32, i32, i32, i32, i32, f32, f32, i32, P(i64)]
    L.ltr_remove_pass_adaptive.argtypes = [vp, i32, i32, i32, i32, i32, i32, f32, f32, i32, P(i64)]
    L.ltr_remove_pass_ball.argtypes = [vp, i32, i32, i32, i32, i32, i32, f32, f32, f32, f32, i32, P(i64)]
    L.ltr_scan_images_release.argtypes = [vp, i32]
    L.ltr_flags_device_ptr.argtypes = [vp, i32, P(vp), P(i64)]
    L.ltr_flags_download.argtypes = [vp, i32, vp, i64]
    L.ltr_flags_upload.argtypes = [vp, i32, vp, i64]
    L.ltr_apply_partition.argtypes = [vp, i32, P(i32), P(i32)]
    L.ltr_parse_projected.argtypes = [vp, i32, i32, i32, i32, f32, P(i32)]
    L.ltr_knn_diff.argtypes = [vp, i32, i32, i32, i32, i32, f32, P(i32), P(i32)]
    L.ltr_knn_split_cloud.argtypes = [vp, i32, i32, i32, f32, P(i32), P(i32)]
    L.ltr_knn_split_per_keyframe.argtypes = [vp, i32, i32, i32, f32, P(i32), P(i32)]
    L.ltr_scanside_split.argtypes = [vp, i32, i32, i32, i32, i32, i32, f32, P(i32), P(i32)]
    L.ltr_scanside_stats.argtypes = [vp, vp]
    L.ltr_icp_params_default.argtypes = [P(IcpParams)]
    L.ltr_icp_params_default.restype = None
    L.ltr_icp_refine.argtypes = [vp, i32, i32, i32, i32, P(IcpParams), vp, vp, vp, vp]
    L.ltr_knn_diff_refined.argtypes = [vp, i32, i32, i32, i32, i32, f32, vp, vp, P(i32), P(i32)]
    L.ltr_icp_refine_scanside.argtypes = [vp, i32, i32, i32, i32, P(IcpParams), vp, vp, vp, vp]
    L.ltr_scanside_split_refined.argtypes = [vp, i32, i32, i32, i32, i32, i32, f32, vp, vp, P(i32), P(i32)]
    L.ltr_debug_pixel_index.argtypes = [vp, vp, i64, i32, i32, vp, vp, vp, vp, vp]
    L.ltr_debug_scan_rimg.argtypes = [vp, i32, i32, ctypes.c_float, vp]
    L.ltr_debug_exact_knn_avg.argtypes = [vp, i32, i32, i32, i32, vp, P(i64)]
    L.ltr_debug_nearest.argtypes = [vp, i32, i32, vp, vp]
    L.ltr_debug_fast_project.argtypes = [vp, vp, i64, vp, f32, vp, vp]
    L.ltr_debug_atan_sweep.argtypes = [vp, i32, P(ctypes.c_double), P(f32)]
    L.ltr_debug_margins.argtypes = [vp, f32, vp]
    L.ltr_debug_voxel_distributed.argtypes = [vp, i32, vp, f32, P(i32), vp, vp]
    L.ltr_reset_rimg_size.argtypes = [f32, f32, f32, P(i32), P(i32)]
    L.ltr_reset_rimg_size.restype = None
    L.ltr_last_pass_stats.argtypes = [vp, vp]
    L.ltr_profile_get.argtypes = [vp, vp]
    L.ltr_profile_reset.argtypes = [vp]
    L.ltr_timer_start.argtypes = [vp]
    L.ltr_trace_dump.argtypes = [vp, i32]
    L.ltr_timer_stop.argtypes = [vp, P(ctypes.c_double)]
    L.ltr_pinned_alloc.argtypes = [ctypes.c_size_t, P(vp)]
    L.ltr_pinned_free.argtypes = [vp]
    L.ltr_pinned_free.restype = None
    L.ltr_nccl_unique_id.argtypes = [vp]
    L.ltr_nccl_init.argtypes = [vp, vp, i32, i32, P(i32)]
    L.ltr_nccl_split.argtypes = [vp, i32, i32, i32, P(i32)]
    L.ltr_nccl_info.argtypes = [vp, i32, P(i32), P(i32)]
    L.ltr_nccl_destroy.argtypes = [vp, i32]
    L.ltr_nccl_version.argtypes = [P(i32)]
    L.ltr_nccl_allreduce_flags.argtypes = [vp, i32, i32]
    L.ltr_nccl_allgather_clouds.argtypes = [vp, i32, i32, vp, vp]
    L.ltr_nccl_voxel_centroid_merged.argtypes = [vp, i32, i32, f32, P(i32)]
    L.ltr_nccl_exchange_clouds.argtypes = [vp, i32, i32, i32, vp, i32, vp]
    L.ltr_nccl_allgather_i64.argtypes = [vp, i32, vp, i32, vp]
    L.ltr_nccl_max_f64.argtypes = [vp, i32, ctypes.c_double, P(ctypes.c_double)]
    L.ltr_nccl_barrier.argtypes = [vp, i32]
    L.ltr_stream_handle.argtypes = [vp]
    L.ltr_stream_handle.restype = vp
    _LIB = L
    return L


def reset_rimg_size(alpha, vfov=50.0, hfov=360.0):
    r, c = ctypes.c_int32(), ctypes.c_int32()
    lib().ltr_reset_rimg_size(vfov, hfov, alpha, ctypes.byref(r), ctypes.byref(c))
    return r.value, c.value


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


class Context:
    """One GPU context (ltr_ctx).  Handles returned by its methods are plain ints."""

    def __init__(self, device=0, vfov=50.0, hfov=360.0, lidar2base=None, base2lidar=None, transform_order=0,
                 keyframe_batch=0, fast_path=True, cull=True):
        L = lib()
        cfg = Config()
        L.ltr_config_default(ctypes.byref(cfg))
        cfg.device = device
        cfg.vfov_deg, cfg.hfov_deg = vfov, hfov
        self._vfov, self._hfov = vfov, hfov
        if lidar2base is not None:
            l2b = np.ascontiguousarray(lidar2base, np.float64).reshape(16)
            b2l = (np.ascontiguousarray(base2lidar, np.float64).reshape(16) if base2lidar is not None
                   else np.linalg.inv(l2b.reshape(4, 4)).reshape(16))
            for i in range(16):
                cfg.lidar2base[i] = l2b[i]
                cfg.base2lidar[i] = b2l[i]
        cfg.transform_order = transform_order
        cfg.keyframe_batch = keyframe_batch
        cfg.fast_path = (2 if cull else 1) if fast_path else 0
        self._h = ctypes.c_void_p()
        rc = L.ltr_create(ctypes.byref(self._h), ctypes.byref(cfg))
        if rc != LTR_OK:
            msg = L.ltr_last_error(None).decode()
            self._h = None
            raise LtrError(rc, msg)

    def close(self):
        if getattr(self, "_h", None):
            lib().ltr_destroy(self._h)
            self._h = None

    def __del__(self):
        self.close()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def _ck(self, rc):
        if rc != LTR_OK:
            raise LtrError(rc, lib().ltr_last_error(self._h).decode())

    # ---- data movement ----
    def cloud_upload(self, xyzi):
        x = _f32(xyzi).reshape(-1, 4)
        h = ctypes.c_int32()
        self._ck(lib().ltr_cloud_upload(self._h, x.ctypes.data, len(x), ctypes.byref(h)))
        return h.value

    def cloud_size(self, c):
        n = ctypes.c_int64()
        self._ck(lib().ltr_cloud_size(self._h, c, ctypes.byref(n)))
        return n.value

    def cloud_download(self, c, out=None):
        """Downloads cloud `c` as (n, 4) float32.  `out` may be a caller-owned (capacity, 4) float32 array (e.g. pinned
        host memory for a fast D2H); the returned array is then a view of its first n rows."""
        n = self.cloud_size(c)
        if out is None:
            out = np.empty((n, 4), np.float32)
        elif out.dtype != np.float32 or out.ndim != 2 or out.shape[1] != 4 or len(out) < n or not out.flags.c_contiguous:
            raise ValueError("out must be a C-contiguous float32 array of shape (>= n, 4)")
        m = ctypes.c_int64()
        self._ck(lib().ltr_cloud_download(self._h, c, out.ctypes.data, len(out), ctypes.byref(m)))
        return out[:n]

    def cloud_free(self, c):
        self._ck(lib().ltr_cloud_free(self._h, c))

    def cloud_copy(self, c):
        h = ctypes.c_int32()
        self._ck(lib().ltr_cloud_copy(self._h, c, ctypes.byref(h)))
        return h.value

    def cloud_concat(self, a, b):
        h = ctypes.c_int32()
        self._ck(lib().ltr_cloud_concat(self._h, a, b, ctypes.byref(h)))
        return h.value

    def cloud_slice(self, c, begin, end):
        """Non-owning view of the points [begin, end) of cloud `c` (ltr_cloud_slice): valid while `c` lives, freed like any cloud."""
        h = ctypes.c_int32()
        self._ck(lib().ltr_cloud_slice(self._h, c, begin, end, ctypes.byref(h)))
        return h.value

    def scanset_upload(self, xyzi, offsets):
        x = _f32(xyzi).reshape(-1, 4)
        o = np.ascontiguousarray(offsets, np.int64)
        h = ctypes.c_int32()
        self._ck(lib().ltr_scanset_upload(self._h, x.ctypes.data, o.ctypes.data, len(o) - 1, ctypes.byref(h)))
        return h.value

    def scanset_info(self, s):
        K, n = ctypes.c_int32(), ctypes.c_int64()
        self._ck(lib().ltr_scanset_info(self._h, s, ctypes.byref(K), ctypes.byref(n)))
        return K.value, n.value

    def scanset_download(self, s):
        K, n = self.scanset_info(s)
        out = np.empty((n, 4), np.float32)
        off = np.empty(K + 1, np.int64)
        self._ck(lib().ltr_scanset_download(self._h, s, out.ctypes.data, n, off.ctypes.data))
        return out, off

    def scanset_free(self, s):
        self._ck(lib().ltr_scanset_free(self._h, s))

    def scanset_concat_per_keyframe(self, a, b):
        h = ctypes.c_int32()
        self._ck(lib().ltr_scanset_concat_per_keyframe(self._h, a, b, ctypes.byref(h)))
        return h.value

    def scanset_flatten(self, s):
        h = ctypes.c_int32()
        self._ck(lib().ltr_scanset_flatten(self._h, s, ctypes.byref(h)))
        return h.value

    def poses_upload(self, poses, inv_poses):
        p = np.ascontiguousarray(poses, np.float64).reshape(-1, 16)
        ip = np.ascontiguousarray(inv_poses, np.float64).reshape(-1, 16)
        assert len(p) == len(ip)
        h = ctypes.c_int32()
        self._ck(lib().ltr_poses_upload(self._h, p.ctypes.data, ip.ctypes.data, len(p), ctypes.byref(h)))
        return h.value

    def poses_free(self, p):
        self._ck(lib().ltr_poses_free(self._h, p))

    # ---- hot path ----
    def preclean(self, scans, radius):
        h = ctypes.c_int32()
        self._ck(lib().ltr_preclean(self._h, scans, radius, ctypes.byref(h)))
        return h.value

    def merge_scans_global(self, scans, poses):
        h = ctypes.c_int32()
        self._ck(lib().ltr_merge_scans_global(self._h, scans, poses, ctypes.byref(h)))
        return h.value

    def voxel_centroid(self, cloud, leaf):
        h = ctypes.c_int32()
        self._ck(lib().ltr_voxel_centroid(self._h, cloud, leaf, ctypes.byref(h)))
        return h.value

    def voxel_centroid_per_keyframe(self, scans, leaf):
        h = ctypes.c_int32()
        self._ck(lib().ltr_voxel_centroid_per_keyframe(self._h, scans, leaf, ctypes.byref(h)))
        return h.value

    def voxel_grid(self, cloud, leaf):
        """Load-time pcl::VoxelGrid of one cloud (ltr_voxel_grid).  Returns (handle, overflowed): overflowed is True when the
        filter took PCL's overflow exit and the output is the input unchanged."""
        h, ov = ctypes.c_int32(), ctypes.c_int32()
        self._ck(lib().ltr_voxel_grid(self._h, cloud, leaf, ctypes.byref(h), ctypes.byref(ov)))
        return h.value, bool(ov.value)

    def voxel_grid_per_keyframe(self, scans, leaf):
        """Load-time pcl::VoxelGrid of every keyframe (ltr_voxel_grid_per_keyframe).  Returns (handle, number of scans returned
        unchanged by the overflow exit)."""
        h, ov = ctypes.c_int32(), ctypes.c_int32()
        self._ck(lib().ltr_voxel_grid_per_keyframe(self._h, scans, leaf, ctypes.byref(h), ctypes.byref(ov)))
        return h.value, ov.value

    def _remove_pass(self, fn, map_, scans, poses, kf_begin, kf_end, mode, res_alpha, thresholds, accumulate):
        """One ltr_remove_pass* call over [kf_begin, kf_end) (kf_end None: every keyframe of `scans`); returns the flagged count."""
        if kf_end is None:
            kf_end = self.scanset_info(scans)[0]
        n = ctypes.c_int64()
        self._ck(fn(self._h, map_, scans, poses, kf_begin, kf_end, mode, res_alpha, *thresholds, 1 if accumulate else 0, ctypes.byref(n)))
        return n.value

    def remove_pass(self, map_, scans, poses, mode, res_alpha, diff_thres=0.1, kf_begin=0, kf_end=None, accumulate=False):
        return self._remove_pass(lib().ltr_remove_pass, map_, scans, poses, kf_begin, kf_end, mode, res_alpha, (diff_thres,), accumulate)

    def remove_pass_adaptive(self, map_, scans, poses, mode, res_alpha, coeff=0.05, kf_begin=0, kf_end=None, accumulate=False):
        """remove_pass with the range-adaptive threshold fl(coeff * scan range) per pixel (ltr_remove_pass_adaptive; 0 < coeff < 1)."""
        return self._remove_pass(lib().ltr_remove_pass_adaptive, map_, scans, poses, kf_begin, kf_end, mode, res_alpha, (coeff,), accumulate)

    def remove_pass_ball(self, map_, scans, poses, mode, res_alpha, radius, diff_thres=0.1, adaptive_coeff=0.0, kf_begin=0, kf_end=None,
                         accumulate=False):
        """remove_pass in which each keyframe sees only the map points within `radius` of its pose's translation (ltr_remove_pass_ball);
        adaptive_coeff != 0 takes the range-adaptive threshold instead of diff_thres."""
        return self._remove_pass(lib().ltr_remove_pass_ball, map_, scans, poses, kf_begin, kf_end, mode, res_alpha,
                                 (diff_thres, adaptive_coeff, radius), accumulate)

    def scan_images_release(self, free_storage=True):
        """Drops the scan-side images remove_pass keeps between passes; free_storage also frees their storage (ltr_scan_images_release)."""
        self._ck(lib().ltr_scan_images_release(self._h, 1 if free_storage else 0))

    def flags_download(self, map_):
        n = self.cloud_size(map_)
        out = np.empty(n, np.uint8)
        self._ck(lib().ltr_flags_download(self._h, map_, out.ctypes.data, n))
        return out

    def flags_upload(self, map_, flags):
        f = np.ascontiguousarray(flags, np.uint8)
        self._ck(lib().ltr_flags_upload(self._h, map_, f.ctypes.data, len(f)))

    def flags_device_ptr(self, map_):
        p, n = ctypes.c_void_p(), ctypes.c_int64()
        self._ck(lib().ltr_flags_device_ptr(self._h, map_, ctypes.byref(p), ctypes.byref(n)))
        return p.value, n.value

    def apply_partition(self, map_):
        s, d = ctypes.c_int32(), ctypes.c_int32()
        self._ck(lib().ltr_apply_partition(self._h, map_, ctypes.byref(s), ctypes.byref(d)))
        return s.value, d.value

    def parse_projected(self, map_, poses, kf_begin, kf_end, res_alpha=3.0):
        h = ctypes.c_int32()
        self._ck(lib().ltr_parse_projected(self._h, map_, poses, kf_begin, kf_end, res_alpha, ctypes.byref(h)))
        return h.value

    def knn_diff(self, scans, poses, target, k, thr, pose_offset=0):
        a, b = ctypes.c_int32(), ctypes.c_int32()
        self._ck(lib().ltr_knn_diff(self._h, scans, poses, pose_offset, target, k, thr, ctypes.byref(a), ctypes.byref(b)))
        return a.value, b.value

    def knn_split_cloud(self, query, target, k, thr):
        a, b = ctypes.c_int32(), ctypes.c_int32()
        self._ck(lib().ltr_knn_split_cloud(self._h, query, target, k, thr, ctypes.byref(a), ctypes.byref(b)))
        return a.value, b.value

    def knn_split_per_keyframe(self, query, target, k, thr):
        """(near, far) scan sets of ltr_knn_split_per_keyframe: keyframe j of `query` against keyframe j of `target`; an empty target
        keyframe makes all its query points far."""
        a, b = ctypes.c_int32(), ctypes.c_int32()
        self._ck(lib().ltr_knn_split_per_keyframe(self._h, query, target, k, thr, ctypes.byref(a), ctypes.byref(b)))
        return a.value, b.value

    def scanside_split(self, scans, poses, map_, criterion, k, thr, pose_offset=0):
        """(static, dynamic) scan sets of ltr_scanside_split."""
        a, b = ctypes.c_int32(), ctypes.c_int32()
        self._ck(lib().ltr_scanside_split(self._h, scans, poses, pose_offset, map_, criterion, k, thr, ctypes.byref(a), ctypes.byref(b)))
        return a.value, b.value

    def icp_refine(self, scans, poses, target_down, pose_offset=0, **params):
        """ltr_icp_refine: per keyframe (T (K, 4, 4) float32, fitness (K,) float64, iterations (K,) int32, exit reason (K,) int32).
        Keyword arguments override fields of ltr_icp_params (defaults: the reference's values), e.g. max_iterations=5."""
        return self._icp(lib().ltr_icp_refine, scans, poses, target_down, pose_offset, params)

    def icp_refine_scanside(self, scans, poses, target_down, pose_offset=0, **params):
        """ltr_icp_refine_scanside: icp_refine with each scan moved to the global frame as scan-side removal moves it (lidar2base)."""
        return self._icp(lib().ltr_icp_refine_scanside, scans, poses, target_down, pose_offset, params)

    def _icp(self, fn, scans, poses, target_down, pose_offset, params):
        prm = IcpParams()
        lib().ltr_icp_params_default(ctypes.byref(prm))
        for key, v in params.items():
            if not hasattr(prm, key):
                raise TypeError(f"unknown ICP parameter {key}")
            setattr(prm, key, v)
        K = self.scanset_info(scans)[0]
        T = np.empty((K, 4, 4), np.float32)
        fit = np.empty(K, np.float64)
        it = np.empty(K, np.int32)
        ex = np.empty(K, np.int32)
        self._ck(fn(self._h, scans, poses, pose_offset, target_down, ctypes.byref(prm), T.ctypes.data, fit.ctypes.data, it.ctypes.data,
                    ex.ctypes.data))
        return T, fit, it, ex

    def knn_diff_refined(self, scans, poses, target, k, thr, T, accepted, pose_offset=0):
        """(coexist, diff) scan sets of ltr_knn_diff_refined: keyframes with accepted[k] are moved by T[k] (float32 4x4) first."""
        K = self.scanset_info(scans)[0]
        Tf = np.ascontiguousarray(T, np.float32).reshape(K * 16)
        acc = np.ascontiguousarray(accepted, np.uint8).reshape(K)
        a, b = ctypes.c_int32(), ctypes.c_int32()
        self._ck(lib().ltr_knn_diff_refined(self._h, scans, poses, pose_offset, target, k, thr, Tf.ctypes.data, acc.ctypes.data,
                                            ctypes.byref(a), ctypes.byref(b)))
        return a.value, b.value

    def scanside_split_refined(self, scans, poses, map_, criterion, k, thr, T, accepted, pose_offset=0):
        """(static, dynamic) scan sets of ltr_scanside_split_refined: keyframes with accepted[k] are moved by T[k] (float32 4x4) first.
        T or accepted None passes NULL."""
        K = self.scanset_info(scans)[0]
        Tf = None if T is None else np.ascontiguousarray(T, np.float32).reshape(K * 16)
        acc = None if accepted is None else np.ascontiguousarray(accepted, np.uint8).reshape(K)
        a, b = ctypes.c_int32(), ctypes.c_int32()
        self._ck(lib().ltr_scanside_split_refined(self._h, scans, poses, pose_offset, map_, criterion, k, thr,
                                                  None if Tf is None else Tf.ctypes.data, None if acc is None else acc.ctypes.data,
                                                  ctypes.byref(a), ctypes.byref(b)))
        return a.value, b.value

    def scanside_stats(self):
        out = np.zeros(4, np.int64)
        self._ck(lib().ltr_scanside_stats(self._h, out.ctypes.data))
        return out

    # ---- introspection ----
    def debug_pixel_index(self, xyz, rows, cols):
        x = _f32(xyz).reshape(-1, 3)
        n = len(x)
        row = np.empty(n, np.int32); col = np.empty(n, np.int32)
        rng = np.empty(n, np.float32); az = np.empty(n, np.float32); el = np.empty(n, np.float32)
        self._ck(lib().ltr_debug_pixel_index(self._h, x.ctypes.data, n, rows, cols, row.ctypes.data, col.ctypes.data,
                                             rng.ctypes.data, az.ctypes.data, el.ctypes.data))
        return row, col, rng, az, el

    def debug_scan_rimg(self, scans, kf, res_alpha):
        rows, cols = reset_rimg_size(res_alpha, self._vfov, self._hfov)
        out = np.empty((rows, cols), np.float32)
        self._ck(lib().ltr_debug_scan_rimg(self._h, scans, kf, res_alpha, out.ctypes.data))
        return out

    def debug_exact_knn_avg(self, query, k, target=None):
        """(avg (n,) float32, unsettled) of ltr_debug_exact_knn_avg: scan set `query` against cloud `target`, or each keyframe of `query`
        against its own points when target is None."""
        n = self.scanset_info(query)[1]
        out = np.empty(n, np.float32)
        un = ctypes.c_int64()
        self._ck(lib().ltr_debug_exact_knn_avg(self._h, query, -1 if target is None else target, 1 if target is None else 0, k,
                                               out.ctypes.data, ctypes.byref(un)))
        return out, un.value

    def debug_nearest(self, query, target):
        """(d (n,) float32, idx (n,) int32) of ltr_debug_nearest: ICP's nearest target point for every point of cloud `query`."""
        n = self.cloud_size(query)
        d = np.empty(n, np.float32)
        idx = np.empty(n, np.int32)
        self._ck(lib().ltr_debug_nearest(self._h, query, target, d.ctypes.data, idx.ctypes.data))
        return d, idx

    def debug_fast_project(self, xyz, inv_pose, res_alpha):
        x = _f32(xyz).reshape(-1, 3)
        ip = np.ascontiguousarray(inv_pose, np.float64).reshape(16)
        out = np.empty((len(x), 8), np.float32)
        mg = np.zeros(4, np.float32)
        self._ck(lib().ltr_debug_fast_project(self._h, x.ctypes.data, len(x), ip.ctypes.data, res_alpha, out.ctypes.data, mg.ctypes.data))
        return out, mg

    def debug_atan_sweep(self, which):
        """(max |poly(a) - atan(a)|, argument) over EVERY float of [0, 1] (which = 0, azimuth polynomial) or [0, 0.5] (which = 1)."""
        e, a = ctypes.c_double(), ctypes.c_float()
        self._ck(lib().ltr_debug_atan_sweep(self._h, which, ctypes.byref(e), ctypes.byref(a)))
        return e.value, a.value

    def debug_margins(self, res_alpha):
        m = np.zeros(9, np.float32)
        self._ck(lib().ltr_debug_margins(self._h, res_alpha, m.ctypes.data))
        return m

    def debug_voxel_distributed(self, locals_, leaf):
        """ltr_debug_voxel_distributed over len(locals_) simulated ranks, rank r holding cloud locals_[r]: (handle of the voxelised
        concatenation, cuts (world - 1,) uint32, send counts (world, world) int64 with [r, d] = points rank r sends to rank d)."""
        G = len(locals_)
        hs = np.ascontiguousarray(locals_, np.int32)
        cuts = np.zeros(max(G - 1, 1), np.uint32)
        sc = np.zeros((max(G, 1), max(G, 1)), np.int64)
        h = ctypes.c_int32()
        self._ck(lib().ltr_debug_voxel_distributed(self._h, G, hs.ctypes.data, leaf, ctypes.byref(h), cuts.ctypes.data, sc.ctypes.data))
        return h.value, cuts[: max(G - 1, 0)], sc[:G, :G]

    def last_pass_stats(self):
        s = np.zeros(7, np.float64)
        self._ck(lib().ltr_last_pass_stats(self._h, s.ctypes.data))
        return s

    def profile_get(self):
        s = np.zeros(8, np.float64)
        self._ck(lib().ltr_profile_get(self._h, s.ctypes.data))
        return s

    def profile_reset(self):
        self._ck(lib().ltr_profile_reset(self._h))

    def trace_dump(self, reset=True):
        self._ck(lib().ltr_trace_dump(self._h, 1 if reset else 0))

    def timer_start(self):
        self._ck(lib().ltr_timer_start(self._h))

    def timer_stop(self):
        ms = ctypes.c_double()
        self._ck(lib().ltr_timer_stop(self._h, ctypes.byref(ms)))
        return ms.value

    def kernel_launches(self):
        return lib().ltr_kernel_launches(self._h)

    def voxel_shortcuts(self):
        return lib().ltr_voxel_shortcuts(self._h)

    def memory_stats(self):
        """(live, cached, peak_live) bytes of the context's caching allocator."""
        s = np.zeros(3, np.int64)
        self._ck(lib().ltr_memory_stats(self._h, s.ctypes.data))
        return tuple(int(v) for v in s)

    def synchronize(self):
        self._ck(lib().ltr_synchronize(self._h))

    def stream_handle(self):
        """cudaStream_t (as int) every kernel and collective of this context runs on."""
        return lib().ltr_stream_handle(self._h)
