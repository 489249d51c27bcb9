"""Python view of the host orchestrator (include/ltr_removert.h, libltr_removert.so).

`Removerter` mirrors ltremovert::Removerter (ltremovert/src/Removerter.cpp:1653-1678): load two sessions,
run Step 0 / Step 1+2 / Step 3, read back named clouds.  All work happens in the C++ orchestrator and the
CUDA library underneath; this module only moves numpy arrays across the C-ABI.  Multi-GPU runs use the
library's native NCCL transport (`Removerter.init_nccl`).
"""
import ctypes
import os

import numpy as np

from . import binding

_HERE = os.path.dirname(os.path.abspath(__file__))
HOST_LIB_PATH = os.path.join(_HERE, "libltr_removert.so")
_LIB = None

OP_REMOVE, OP_REVERT = 0, 1
MAX_SCHEDULE = 32


class Params(ctypes.Structure):
    _fields_ = [("device", ctypes.c_int32), ("sequence_vfov", ctypes.c_float), ("sequence_hfov", ctypes.c_float),
                ("ExtrinsicLiDARtoPoseBase", ctypes.c_double * 16), ("num_nn_points_within", ctypes.c_int32),
                ("dist_nn_points_within", ctypes.c_float), ("downsample_voxel_size", ctypes.c_float),
                ("n_schedule", ctypes.c_int32), ("schedule_op", ctypes.c_int32 * MAX_SCHEDULE),
                ("schedule_res", ctypes.c_float * MAX_SCHEDULE), ("extract_high_dyn_knn", ctypes.c_int32),
                ("transform_order", ctypes.c_int32), ("keyframe_batch", ctypes.c_int32), ("fast_path", ctypes.c_int32)]


HOST_EXPORTS = ["ltrh_params_default", "ltrh_create", "ltrh_destroy", "ltrh_last_error", "ltrh_context", "ltrh_comm_init_nccl", "ltrh_owns_session", "ltrh_invert_poses",
                "ltrh_load_session", "ltrh_load_session_raw", "ltrh_run_step0", "ltrh_run_step12", "ltrh_run_step3", "ltrh_reset_to_step0", "ltrh_cascade_promote_updated", "ltrh_set_delta_maps", "ltrh_delta_load", "ltrh_delta_count", "ltrh_compose_changes", "ltrh_rollback", "ltrh_scanside_removal", "ltrh_scanside_removal_registered", "ltrh_set_icp_refinement", "ltrh_set_adaptive_threshold", "ltrh_set_map_ball", "ltrh_icp_stats", "ltrh_scanside_icp_stats", "ltrh_stage", "ltrh_cloud",
                "ltrh_scanset", "ltrh_timing", "ltrh_log_count", "ltrh_log_get", "ltrh_io_last_error", "ltrh_io_read_pcd", "ltrh_io_write_pcd",
                "ltrh_io_read_poses", "ltrh_io_parse_keyframes", "ltrh_io_parse_keyframes_in_roi", "ltrh_io_voxel_grid", "ltrh_io_voxel_grid_scans", "ltrh_io_yaml_get"]


def host_lib():
    global _LIB
    if _LIB is not None:
        return _LIB
    binding.lib()  # the device library must be loadable first (fails loudly if it has not been built)
    if not os.path.exists(HOST_LIB_PATH):
        raise ImportError(f"{HOST_LIB_PATH} is missing: run __graft_entry__.build()")
    L = ctypes.CDLL(HOST_LIB_PATH)
    vp, i32, i64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64
    P = ctypes.POINTER
    L.ltrh_params_default.argtypes = [P(Params)]
    L.ltrh_params_default.restype = None
    L.ltrh_create.argtypes = [P(vp), P(Params)]
    L.ltrh_destroy.argtypes = [vp]
    L.ltrh_destroy.restype = None
    L.ltrh_last_error.argtypes = [vp]
    L.ltrh_last_error.restype = ctypes.c_char_p
    L.ltrh_context.argtypes = [vp]
    L.ltrh_context.restype = vp
    L.ltrh_comm_init_nccl.argtypes = [vp, vp, i32, i32, i32]
    L.ltrh_owns_session.argtypes = [vp, i32]
    L.ltrh_invert_poses.argtypes = [vp, i32, vp]
    L.ltrh_invert_poses.restype = None
    L.ltrh_load_session.argtypes = [vp, i32, vp, vp, vp, vp, i32]
    L.ltrh_load_session_raw.argtypes = [vp, i32, vp, vp, vp, vp, i32]
    for f in ("ltrh_run_step0", "ltrh_run_step12", "ltrh_run_step3", "ltrh_reset_to_step0", "ltrh_cascade_promote_updated"):
        getattr(L, f).argtypes = [vp]
    L.ltrh_set_delta_maps.argtypes = [vp, i32]
    L.ltrh_delta_load.argtypes = [vp, vp, vp, vp, vp]
    L.ltrh_delta_count.argtypes = [vp]
    L.ltrh_compose_changes.argtypes = [vp, i32, i32]
    L.ltrh_rollback.argtypes = [vp, i32]
    L.ltrh_scanside_removal.argtypes = [vp, i32, i32, i32]
    L.ltrh_scanside_removal_registered.argtypes = [vp, i32, i32, i32]
    L.ltrh_set_icp_refinement.argtypes = [vp, i32]
    L.ltrh_set_adaptive_threshold.argtypes = [vp, ctypes.c_float]
    L.ltrh_set_map_ball.argtypes = [vp, ctypes.c_float]
    L.ltrh_icp_stats.argtypes = [vp, i32, i32, P(i32), vp, vp, vp, vp, vp]
    L.ltrh_scanside_icp_stats.argtypes = [vp, i32, i32, P(i32), vp, vp, vp, vp, vp]
    L.ltrh_stage.argtypes = [vp, ctypes.c_char_p]
    L.ltrh_cloud.argtypes = [vp, ctypes.c_char_p, i32, P(i32)]
    L.ltrh_scanset.argtypes = [vp, ctypes.c_char_p, i32, P(i32)]
    L.ltrh_timing.argtypes = [vp, ctypes.c_char_p]
    L.ltrh_timing.restype = ctypes.c_double
    L.ltrh_log_count.argtypes = [vp]
    L.ltrh_log_get.argtypes = [vp, i32, ctypes.c_char_p, i32, vp]
    L.ltrh_io_last_error.restype = ctypes.c_char_p
    L.ltrh_io_read_pcd.argtypes = [ctypes.c_char_p, vp, i64]
    L.ltrh_io_read_pcd.restype = i64
    L.ltrh_io_write_pcd.argtypes = [ctypes.c_char_p, vp, i64, i32]
    L.ltrh_io_read_poses.argtypes = [ctypes.c_char_p, vp, i32]
    L.ltrh_io_parse_keyframes.argtypes = [i32, i32, i32, i32, vp, i32]
    L.ltrh_io_parse_keyframes_in_roi.argtypes = [vp, i32, vp, i32, i32, vp, i32]
    L.ltrh_io_voxel_grid.argtypes = [vp, i64, ctypes.c_float, vp, i64, P(i32)]
    L.ltrh_io_voxel_grid.restype = i64
    L.ltrh_io_voxel_grid_scans.argtypes = [vp, vp, i32, ctypes.c_float, vp, i64, vp]
    L.ltrh_io_voxel_grid_scans.restype = i64
    L.ltrh_io_yaml_get.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_char_p, i32, vp, i32, P(i32)]
    _LIB = L
    return L


def inverse_poses(poses):
    """Inverse keyframe poses as the reference computes them (general 4x4 cofactor inverse, Session.cpp:110); np.linalg.inv differs in the
    last bits, which is enough to move a few emitted coordinates by one ulp."""
    p = np.ascontiguousarray(poses, np.float64).reshape(-1, 4, 4)
    out = np.empty_like(p)
    host_lib().ltrh_invert_poses(p.ctypes.data, len(p), out.ctypes.data)
    return out


def nccl_unique_id():
    """128 bytes of ncclGetUniqueId (call on ONE rank, hand the bytes to the others through the launcher's own channel)."""
    buf = ctypes.create_string_buffer(128)
    rc = binding.lib().ltr_nccl_unique_id(buf)
    if rc != 0:
        raise binding.LtrError(rc, binding.lib().ltr_last_error(None).decode())
    return bytes(buf.raw)


def selfremovert_schedule(resolutions):
    """Removerter::selfRemovert (Removerter.cpp:1378-1393): remove(r), revert(0.95 r), remove(r) per resolution.  The revert
    resolution is `0.95 * _res_alpha` with a float argument, i.e. a DOUBLE product narrowed once when passed on as float (:1385)."""
    s = []
    for r in resolutions:
        s += [(OP_REMOVE, r), (OP_REVERT, float(np.float32(0.95 * float(np.float32(r))))), (OP_REMOVE, r)]
    return s


class Removerter:
    def __init__(self, device=0, vfov=50.0, hfov=360.0, lidar2base=None, num_knn=2, knn_thr=0.01, voxel=0.05,
                 schedule=((OP_REMOVE, 2.5),), extract_high_dyn_knn=True, transform_order=0, keyframe_batch=0,
                 fast_path=True, cull=True):
        L = host_lib()
        p = Params()
        L.ltrh_params_default(ctypes.byref(p))
        p.device = device
        p.sequence_vfov, p.sequence_hfov = vfov, hfov
        if lidar2base is not None:
            l2b = np.ascontiguousarray(lidar2base, np.float64).reshape(16)
            for i in range(16):
                p.ExtrinsicLiDARtoPoseBase[i] = l2b[i]
        p.num_nn_points_within, p.dist_nn_points_within, p.downsample_voxel_size = num_knn, knn_thr, voxel
        schedule = list(schedule)
        p.n_schedule = len(schedule)
        for i, (op, res) in enumerate(schedule):
            p.schedule_op[i], p.schedule_res[i] = op, res
        p.extract_high_dyn_knn = int(extract_high_dyn_knn)
        p.transform_order, p.keyframe_batch, p.fast_path = transform_order, keyframe_batch, ((2 if cull else 1) if fast_path else 0)
        self._h = ctypes.c_void_p()
        rc = L.ltrh_create(ctypes.byref(self._h), ctypes.byref(p))
        if rc != 0:
            msg = L.ltrh_last_error(None).decode()
            self._h = None
            raise binding.LtrError(rc, msg)
        # a binding.Context view that shares the orchestrator's ltr_ctx (not owned)
        self.ctx = binding.Context.__new__(binding.Context)
        self.ctx._h = ctypes.c_void_p(L.ltrh_context(self._h))
        self.K = [0, 0]

    def init_nccl(self, id128, rank, world, split_sessions=True):
        """Native multi-GPU transport (ltrh_comm_init_nccl): every rank passes the same 128-byte id (nccl_unique_id() of one rank)."""
        self._ck(host_lib().ltrh_comm_init_nccl(self._h, id128, rank, world, 1 if split_sessions else 0))

    def owns(self, sess):
        return bool(host_lib().ltrh_owns_session(self._h, sess))

    def close(self):
        if getattr(self, "_h", None):
            self.ctx._h = None
            try:
                host_lib().ltrh_destroy(self._h)
            except TypeError:  # interpreter shutdown
                pass
            self._h = None

    def __del__(self):
        self.close()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def _ck(self, rc):
        if rc != 0:
            raise binding.LtrError(rc, host_lib().ltrh_last_error(self._h).decode())

    def _load(self, fn, sess, xyzi, offsets, poses, inv_poses):
        x = np.ascontiguousarray(xyzi, np.float32)
        o = np.ascontiguousarray(offsets, np.int64)
        p = np.ascontiguousarray(poses, np.float64)
        ip = np.ascontiguousarray(inv_poses, np.float64)
        self._ck(fn(self._h, sess, x.ctypes.data, o.ctypes.data, p.ctypes.data, ip.ctypes.data, len(o) - 1))
        self.K[sess] = len(o) - 1

    def load_session(self, sess, xyzi, offsets, poses, inv_poses):
        self._load(host_lib().ltrh_load_session, sess, xyzi, offsets, poses, inv_poses)

    def load_session_raw(self, sess, xyzi, offsets, poses, inv_poses):
        """load_session from the scans as read from disk: the load-time VoxelGrid at `voxel` runs on the device first
        (ltrh_load_session_raw, Session::loadKeyframes)."""
        self._load(host_lib().ltrh_load_session_raw, sess, xyzi, offsets, poses, inv_poses)

    def run_step0(self):
        self._ck(host_lib().ltrh_run_step0(self._h))

    def run_step12(self):
        self._ck(host_lib().ltrh_run_step12(self._h))

    def run_step3(self):
        self._ck(host_lib().ltrh_run_step3(self._h))

    def reset_to_step0(self):
        self._ck(host_lib().ltrh_reset_to_step0(self._h))

    def cascade_promote_updated(self):
        """LT-map cascade: the updated scans become the central session of the next run (ltrh_cascade_promote_updated)."""
        self._ck(host_lib().ltrh_cascade_promote_updated(self._h))

    def set_delta_maps(self, on=True):
        """LT-map delta maps (ltrh_set_delta_maps): later cascade promotions record each generation's (PD, strong ND) per keyframe; off
        (the default) frees what was recorded."""
        self._ck(host_lib().ltrh_set_delta_maps(self._h, 1 if on else 0))

    def delta_load(self, pd_xyzi, pd_offsets, nd_xyzi, nd_offsets):
        """Appends one generation's delta from arrays (ltrh_delta_load), offsets over this rank's central keyframes."""
        pd = np.ascontiguousarray(pd_xyzi, np.float32).reshape(-1, 4); po = np.ascontiguousarray(pd_offsets, np.int64)
        nd = np.ascontiguousarray(nd_xyzi, np.float32).reshape(-1, 4); no = np.ascontiguousarray(nd_offsets, np.int64)
        self._ck(host_lib().ltrh_delta_load(self._h, pd.ctypes.data, po.ctypes.data, nd.ctypes.data, no.ctypes.data))

    def delta_count(self):
        return host_lib().ltrh_delta_count(self._h)

    def compose_changes(self, i, j):
        """Changes from generation i to j (ltrh_compose_changes): fills the central scan sets "composed_pd_" / "composed_nd_"."""
        self._ck(host_lib().ltrh_compose_changes(self._h, i, j))

    def rollback(self, i):
        """The central scans as of generation i (ltrh_rollback): fills the scan set "keyframe_scans_restored_" and the cloud
        "saved:restored_map"."""
        self._ck(host_lib().ltrh_rollback(self._h, i))

    def scanside_removal(self, map_sess, scan_sess, criterion=0):
        """scansideRemovalForEachScan (ltrh_scanside_removal): fills the scan sets "scans_static_" / "scans_dynamic_" of scan_sess."""
        self._ck(host_lib().ltrh_scanside_removal(self._h, map_sess, scan_sess, criterion))

    def scanside_removal_registered(self, map_sess, scan_sess, criterion=0):
        """scansideRemovalForEachScan with isFineRegistration (ltrh_scanside_removal_registered): every keyframe of scan_sess is registered
        to map_sess's static map at 0.4 m first; fills "scans_static_" / "scans_dynamic_" of scan_sess and scanside_icp_stats(scan_sess)."""
        self._ck(host_lib().ltrh_scanside_removal_registered(self._h, map_sess, scan_sess, criterion))

    def set_icp_refinement(self, on=True):
        """Session::partitionLowDynamicPointsOfScanByKnn's ICP refinement for later Step 2 runs (ltrh_set_icp_refinement; off by default)."""
        self._ck(host_lib().ltrh_set_icp_refinement(self._h, 1 if on else 0))

    def set_adaptive_threshold(self, c=0.05):
        """The range-adaptive threshold fl(c * scan range) for later remove / revert / ND / PD passes (ltrh_set_adaptive_threshold;
        0 < c < 1, c = 0 turns it off, which is the default)."""
        self._ck(host_lib().ltrh_set_adaptive_threshold(self._h, c))

    def set_map_ball(self, radius=80.0):
        """The reference's ball subset of the map for later removeOnce / revertOnce passes (ltrh_set_map_ball): each keyframe projects
        only the map points within `radius` m of its pose; radius = 0 turns it off, which is the default."""
        self._ck(host_lib().ltrh_set_map_ball(self._h, radius))

    def icp_stats(self, sess):
        """This rank's refinement of session `sess` in the last Step 2 (ltrh_icp_stats): dict of per-keyframe arrays T (K, 4, 4) float32,
        fitness, iterations, exit (ltr_icp_exit) and accepted (bool); K = 0 when the step ran without refinement."""
        return self._icp_stats(host_lib().ltrh_icp_stats, sess)

    def scanside_icp_stats(self, sess):
        """The same for the registration of the last scan-side removal of session `sess`'s scans (ltrh_scanside_icp_stats); K = 0 when
        it ran without registration."""
        return self._icp_stats(host_lib().ltrh_scanside_icp_stats, sess)

    def _icp_stats(self, fn, sess):
        K = ctypes.c_int32()
        self._ck(fn(self._h, sess, 0, ctypes.byref(K), None, None, None, None, None))
        n = K.value
        T = np.empty((n, 4, 4), np.float32); fit = np.empty(n, np.float64); it = np.empty(n, np.int32); ex = np.empty(n, np.int32)
        acc = np.empty(n, np.uint8)
        if n:
            self._ck(fn(self._h, sess, n, ctypes.byref(K), T.ctypes.data, fit.ctypes.data, it.ctypes.data, ex.ctypes.data, acc.ctypes.data))
        return {"T": T, "fitness": fit, "iterations": it, "exit": ex, "accepted": acc.astype(bool)}

    def stage(self, name):
        self._ck(host_lib().ltrh_stage(self._h, name.encode()))

    def cloud_handle(self, name, sess=0):
        h = ctypes.c_int32()
        self._ck(host_lib().ltrh_cloud(self._h, name.encode(), sess, ctypes.byref(h)))
        return h.value

    def scanset_handle(self, name, sess=0):
        h = ctypes.c_int32()
        self._ck(host_lib().ltrh_scanset(self._h, name.encode(), sess, ctypes.byref(h)))
        return h.value

    def cloud(self, name, sess=0, out=None):
        return self.ctx.cloud_download(self.cloud_handle(name, sess), out=out)

    def cloud_size(self, name, sess=0):
        return self.ctx.cloud_size(self.cloud_handle(name, sess))

    def scanset(self, name, sess=0):
        return self.ctx.scanset_download(self.scanset_handle(name, sess))

    def timing(self, key):
        return host_lib().ltrh_timing(self._h, key.encode())

    def log(self):
        out = []
        for i in range(host_lib().ltrh_log_count(self._h)):
            buf = ctypes.create_string_buffer(64)
            vals = np.zeros(4, np.int64)
            host_lib().ltrh_log_get(self._h, i, buf, 64, vals.ctypes.data)
            out.append((buf.value.decode(), *[int(v) for v in vals]))
        return out


# ---- file-level helpers (include/ltr_removert.h ltrh_io_*): thin ctypes views used by tests and tools ----
def read_pcd(path):
    L = host_lib()
    n = L.ltrh_io_read_pcd(path.encode(), None, 0)
    if n < 0:
        raise IOError(L.ltrh_io_last_error().decode())
    out = np.empty((n, 4), np.float32)
    L.ltrh_io_read_pcd(path.encode(), out.ctypes.data, n)
    return out


def write_pcd(path, xyzi, octree_layout=False):
    x = np.ascontiguousarray(xyzi, np.float32).reshape(-1, 4)
    if host_lib().ltrh_io_write_pcd(path.encode(), x.ctypes.data, len(x), int(octree_layout)) != 0:
        raise IOError(host_lib().ltrh_io_last_error().decode())


def read_poses(path):
    L = host_lib()
    n = L.ltrh_io_read_poses(path.encode(), None, 0)
    if n < 0:
        raise IOError(L.ltrh_io_last_error().decode())
    out = np.empty((n, 4, 4), np.float64)
    L.ltrh_io_read_poses(path.encode(), out.ctypes.data, n)
    return out


def parse_keyframes(num_scans, start_idx, end_idx, gap):
    out = np.empty(max(num_scans, 1), np.int32)
    n = host_lib().ltrh_io_parse_keyframes(num_scans, start_idx, end_idx, gap, out.ctypes.data, len(out))
    return out[:n].copy()


def parse_keyframes_in_roi(scan_poses, roi_poses, gap):
    a = np.ascontiguousarray(scan_poses, np.float64).reshape(-1, 16)
    b = np.ascontiguousarray(roi_poses, np.float64).reshape(-1, 16)
    out = np.empty(max(len(a), 1), np.int32)
    n = host_lib().ltrh_io_parse_keyframes_in_roi(a.ctypes.data, len(a), b.ctypes.data, len(b), gap, out.ctypes.data, len(out))
    return out[:n].copy()


def voxel_grid(xyzi, leaf):
    x = np.ascontiguousarray(xyzi, np.float32).reshape(-1, 4)
    out = np.empty((max(len(x), 1), 4), np.float32)
    ov = ctypes.c_int32()
    n = host_lib().ltrh_io_voxel_grid(x.ctypes.data, len(x), leaf, out.ctypes.data, len(out), ctypes.byref(ov))
    return out[:n].copy(), bool(ov.value)


def voxel_grid_scans(xyzi, offsets, leaf):
    """The load-time filter over all scans of a session at once (scan k = rows [offsets[k], offsets[k+1])).  Returns (points, offsets)."""
    x = np.ascontiguousarray(xyzi, np.float32).reshape(-1, 4)
    off = np.ascontiguousarray(offsets, np.int64)
    K = len(off) - 1
    out_off = np.zeros(K + 1, np.int64)
    out = np.empty((max(len(x), 1), 4), np.float32)     # the filter never grows a scan
    n = host_lib().ltrh_io_voxel_grid_scans(x.ctypes.data, off.ctypes.data, K, leaf, out.ctypes.data, len(out), out_off.ctypes.data)
    if n < 0:
        raise ValueError("ltrh_io_voxel_grid_scans: bad argument")
    return out[:n].copy(), out_off


def yaml_get(path, key):
    buf = ctypes.create_string_buffer(4096)
    lst = np.zeros(64, np.float64)
    n = ctypes.c_int32()
    if host_lib().ltrh_io_yaml_get(path.encode(), key.encode(), buf, 4096, lst.ctypes.data, 64, ctypes.byref(n)) != 0:
        raise IOError(host_lib().ltrh_io_last_error().decode())
    return buf.value.decode(), lst[:n.value].copy()
