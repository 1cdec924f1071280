"""ctypes binding of the low-level engine C-ABI (include/msckf_b200.h) -- used by bench.py to time the
kernel launch with inputs already resident in HBM, and by tests that exercise the C-ABI directly."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import lib_path

MARGINALIZE, TRIANGULATE, RESIDUALIZE = 0, 1, 2


class Config(C.Structure):
    _fields_ = [("dtype", C.c_int), ("device", C.c_int), ("max_clones", C.c_int), ("max_tracks", C.c_int), ("max_obs", C.c_int)]


class Tracks(C.Structure):
    _fields_ = [("n_tracks", C.c_int), ("obs_offset", C.POINTER(C.c_int)), ("obs", C.c_void_p),
                ("clone_index", C.POINTER(C.c_int)), ("p_f_G", C.c_void_p)]


class Report(C.Structure):
    _fields_ = [("cm_ok", C.POINTER(C.c_int)), ("tri_ok", C.POINTER(C.c_int)), ("valid", C.POINTER(C.c_int)),
                ("accepted", C.POINTER(C.c_int)), ("gamma", C.c_void_p), ("p_f_G", C.c_void_p), ("m", C.c_int), ("rank", C.c_int)]


class NeesResult(C.Structure):
    _fields_ = [("orientation", C.c_double), ("position", C.c_double), ("pose", C.c_double), ("imu", C.c_double),
                ("full", C.c_double), ("dim_full", C.c_int), ("first_bad_pivot", C.c_int)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


def _truth(truth_imu, truth_poses):
    """(19 doubles: p, v, b_g, b_a, g, q_IG xyzw; [M, 7] doubles p_C_G, q_CG xyzw or None) as contiguous float64 arrays"""
    imu = np.ascontiguousarray(truth_imu, dtype=np.float64).ravel()
    assert imu.size == 19, imu.size
    poses = None if truth_poses is None else np.ascontiguousarray(truth_poses, dtype=np.float64).reshape(-1, 7)
    return imu, poses


AID_VELOCITY, AID_POSITION, AID_POSE, AID_CLONE_POSE, AID_LINEAR, AID_BODY_VELOCITY, AID_RELATIVE_POSE = range(7)
AID_ANTENNA_POSITION, AID_CLONE_ANTENNA_POSITION, AID_HEADING, AID_CLONE_HEADING = range(7, 11)
AID_RANGE, AID_CLONE_RANGE, AID_PLANE_RANGE, AID_CLONE_PLANE_RANGE = range(11, 15)
AID_GYRO_AT_REST, AID_ACCEL_AT_REST = 15, 16


class Aid(C.Structure):
    _fields_ = [("model", C.c_int), ("clone", C.c_int), ("m", C.c_int), ("n", C.c_int), ("z", C.c_void_p), ("H", C.c_void_p),
                ("R", C.c_void_p), ("chi2_max", C.c_double)]


class AidResult(C.Structure):
    _fields_ = [("nis", C.c_double), ("dx_norm", C.c_double), ("dof", C.c_int), ("applied", C.c_int), ("status", C.c_int)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


def aid_struct(spec):
    """(Aid, the float64 arrays it points into) of one aided measurement: spec = None (a batch member left alone) or a dict
    model, z (LINEAR: the residual r), R [m, m], H [m, n] (LINEAR), clone (CLONE_POSE), chi2_max"""
    if spec is None or spec["model"] < 0:
        return Aid(-1, 0, 0, 0, None, None, None, 0.0), ()
    z = np.ascontiguousarray(spec["z"], dtype=np.float64).ravel()
    R = np.ascontiguousarray(spec["R"], dtype=np.float64)
    H = None if spec.get("H") is None else np.ascontiguousarray(spec["H"], dtype=np.float64)
    m, n = (H.shape[0], H.shape[1]) if H is not None else (R.shape[0], 0)
    a = Aid(int(spec["model"]), int(spec.get("clone", 0)), m, n, z.ctypes.data, None if H is None else H.ctypes.data,
            R.ctypes.data, float(spec.get("chi2_max", 0.0)))
    return a, (z, R, H)


class AidItem(C.Structure):
    _fields_ = [("model", C.c_int), ("a", C.c_int), ("b", C.c_int), ("z", C.c_void_p), ("R", C.c_void_p)]


def aid_items(items):
    """(AidItem array, the float64 arrays it points into) of one stack: items = list of dicts model, z, R [rows, rows],
    a (CLONE_POSE, RELATIVE_POSE, CLONE_ANTENNA_POSITION and CLONE_HEADING: a clone's window position, BODY_VELOCITY and
    ANTENNA_POSITION: the row mask; "clone" is read when "a" is missing), b (RELATIVE_POSE: the second clone,
    CLONE_ANTENNA_POSITION: the row mask).  z: ANTENNA_POSITION and CLONE_ANTENNA_POSITION p_A_G (3) and the lever arm (3) in
    the body frame, HEADING and CLONE_HEADING psi (1) and the axis (3) in the body frame, RANGE and CLONE_RANGE rho (1), the
    anchor (3) in G and the lever arm (3) in the body frame, PLANE_RANGE and CLONE_PLANE_RANGE rho (1), the plane height h (1),
    the lever arm (3) and the beam axis (3) in the body frame, GYRO_AT_REST the mean gyro reading (3) and ACCEL_AT_REST the
    mean specific force (3) of a standstill (include/msckf_b200.h); "a" of CLONE_RANGE and CLONE_PLANE_RANGE is the clone; R of
    a heading or a range is 1 x 1"""
    arr = (AidItem * max(len(items), 1))()
    keep = []
    for k, it in enumerate(items):
        z = np.ascontiguousarray(it["z"], dtype=np.float64).ravel()
        R = np.ascontiguousarray(it["R"], dtype=np.float64)
        keep += [z, R]
        arr[k] = AidItem(int(it["model"]), int(it.get("a", it.get("clone", 0))), int(it.get("b", 0)), z.ctypes.data, R.ctypes.data)
    return arr, keep


class AidFde(C.Structure):
    _fields_ = [("chi2", C.c_double * 32), ("max_exclude", C.c_int)]


class AidItemResult(C.Structure):
    _fields_ = [("nis", C.c_double), ("test", C.c_double), ("state", C.c_int), ("round", C.c_int)]


class AidFdeResult(C.Structure):
    _fields_ = [("stack", AidResult), ("outcome", C.c_int), ("n_excluded", C.c_int), ("item", AidItemResult * 8)]

    def as_dict(self, n_items):
        d = self.stack.as_dict()
        d.update(outcome=self.outcome, n_excluded=self.n_excluded,
                 items=[{k: getattr(self.item[j], k) for k, _ in AidItemResult._fields_} for j in range(n_items)])
        return d


class AidIter(C.Structure):
    _fields_ = [("max_iter", C.c_int), ("tol", C.c_double)]


class AidIterResult(C.Structure):
    _fields_ = [("iterations", C.c_int), ("converged", C.c_int), ("step", C.c_double)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


def aid_iter_structs(n, max_iter, tol):
    """n msckf_b200_aid_iter of max_iter / tol, each a number or a sequence of n (None: 0)"""
    per = lambda v: list(v) if isinstance(v, (list, tuple, np.ndarray)) else [v] * n  # noqa: E731
    mi, tl = per(max_iter), per(tol)
    assert len(mi) == n and len(tl) == n
    return (AidIter * n)(*[AidIter(int(a or 0), float(b or 0.0)) for a, b in zip(mi, tl)])


def fde_thresholds(alpha):
    """chi2[d - 1] = the chi-square quantile 1 - alpha of d dof, d = 1..32 (the thresholds of msckf_b200_aid_fde)"""
    from scipy.stats import chi2
    return [float(chi2.ppf(1.0 - alpha, d)) for d in range(1, 33)]


def fde_struct(fde):
    """msckf_b200_aid_fde of fde = dict chi2 (32 thresholds, chi2[d - 1] for d rows; see fde_thresholds), max_exclude (0..7)"""
    chi2 = np.asarray(fde["chi2"], dtype=np.float64).ravel()
    assert chi2.size == 32, chi2.size
    return AidFde((C.c_double * 32)(*chi2.tolist()), int(fde["max_exclude"]))


class Standstill(C.Structure):
    _fields_ = [("noise_scale", C.c_double), ("sigma_v", C.c_double), ("scatter_max", C.c_double), ("chi2_max", C.c_double)]


class StandstillResult(C.Structure):
    _fields_ = [("stack", AidResult), ("scatter", C.c_double), ("outcome", C.c_int)]

    def as_dict(self):
        d = self.stack.as_dict()
        d.update(scatter=self.scatter, outcome=self.outcome)
        return d


def standstill_struct(cfg):
    """msckf_b200_standstill of cfg = dict noise_scale (>= 1; default 1), sigma_v (m/s), scatter_max (the largest scatter /
    (6 (k - 1)) taken as at rest), chi2_max (the gate on the 9-row stack's NIS)"""
    return Standstill(float(cfg.get("noise_scale", 1.0)), float(cfg["sigma_v"]), float(cfg["scatter_max"]), float(cfg["chi2_max"]))


class Landmarks(C.Structure):
    _fields_ = [("n_obs", C.c_int), ("clone", C.c_void_p), ("z", C.c_void_p), ("p_L_G", C.c_void_p), ("R", C.c_void_p),
                ("chi2_obs", C.c_double), ("gamma", C.c_void_p), ("flag", C.c_void_p), ("max_iter", C.c_int), ("tol", C.c_double)]


class LandmarkMap(C.Structure):
    _fields_ = [("landmark", C.c_void_p), ("Sigma_L", C.c_void_p), ("n_landmarks", C.c_int)]


class LandmarkResult(C.Structure):
    _fields_ = [("nis", C.c_double), ("dx_norm", C.c_double), ("dof", C.c_int), ("rows", C.c_int), ("used", C.c_int),
                ("applied", C.c_int), ("status", C.c_int), ("iterations", C.c_int), ("converged", C.c_int), ("step", C.c_double)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


def landmark_struct(spec):
    """(Landmarks, the arrays it points into) of one call's mapped-landmark observations: spec = None (a batch member left
    alone) or a dict clone [n] (window positions), z [n, 2], p_L [n, 3], R (None: the filter's pixel noise, else 2 x 2 or
    (uu, uv, vv)), chi2_obs, and optionally max_iter (0 or 1: one linearisation; up to 16: the iterated update) and tol.  The
    arrays are (clone, z, p_L, R, gamma [n] out, flag [n] out)."""
    if spec is None or len(spec["clone"]) == 0:
        return Landmarks(0, None, None, None, None, 0.0, None, None), ()
    clone = np.ascontiguousarray(spec["clone"], dtype=np.int32).ravel()
    z = np.ascontiguousarray(spec["z"], dtype=np.float64).reshape(-1, 2)
    p = np.ascontiguousarray(spec["p_L"], dtype=np.float64).reshape(-1, 3)
    R = spec.get("R")
    if R is not None:
        R = np.asarray(R, dtype=np.float64)
        R = np.ascontiguousarray([R[0, 0], R[1, 0], R[1, 1]] if R.shape == (2, 2) else R.ravel())
    n = len(clone)
    gamma, flag = np.zeros(n), np.zeros(n, dtype=np.int32)
    a = Landmarks(n, clone.ctypes.data, z.ctypes.data, p.ctypes.data, None if R is None else R.ctypes.data,
                  float(spec.get("chi2_obs", 0.0)), gamma.ctypes.data, flag.ctypes.data, int(spec.get("max_iter", 0)),
                  float(spec.get("tol", 0.0)))
    return a, (clone, z, p, R, gamma, flag)


def landmark_map_struct(spec):
    """(LandmarkMap, the arrays it points into) of a spec's map uncertainty: landmark [n] (the landmark of each observation)
    with Sigma_L [n_landmarks, 3, 3] or [n_landmarks, 6] (lower triangle xx, yx, yy, zx, zy, zz).  No Sigma_L (or spec None):
    an exact map, all fields zero."""
    S = None if spec is None else spec.get("Sigma_L")
    if S is None:
        return LandmarkMap(None, None, 0), ()
    lm = spec.get("landmark")
    lm = None if lm is None else np.ascontiguousarray(lm, dtype=np.int32).ravel()
    S = np.asarray(S, dtype=np.float64)
    if S.ndim == 3:
        S = S[:, [0, 1, 1, 2, 2, 2], [0, 0, 1, 0, 1, 2]]
    S = np.ascontiguousarray(S.reshape(-1, 6))
    return LandmarkMap(None if lm is None else lm.ctypes.data, S.ctypes.data, len(S)), (lm, S)


class LandmarkConsensus(C.Structure):
    _fields_ = [("hypotheses", C.c_int), ("thresh", C.c_double), ("min_inliers", C.c_int), ("seed", C.c_ulonglong),
                ("scores", C.c_void_p)]


class LandmarkConsensusResult(C.Structure):
    _fields_ = [("status", C.c_int), ("inliers", C.c_int), ("best", C.c_int), ("valid", C.c_int), ("refit", C.c_int),
                ("yaw", C.c_double), ("t", C.c_double * 3), ("pivot", C.c_double * 3)]

    def as_dict(self, scores=None):
        d = {k: getattr(self, k) for k in ("status", "inliers", "best", "valid", "refit", "yaw")}
        d.update(t=np.array(self.t[:]), pivot=np.array(self.pivot[:]), scores=scores)
        return d


def consensus_struct(cons):
    """(LandmarkConsensus, the arrays it points into) of cons = None (no consensus) or a dict hypotheses (0..1024), thresh,
    min_inliers, seed; the arrays are (scores [hypotheses] out,)"""
    if cons is None or int(cons.get("hypotheses", 0)) == 0:
        return LandmarkConsensus(0, 0.0, 0, 0, None), ()
    h = int(cons["hypotheses"])
    scores = np.zeros(max(h, 0), dtype=np.int32)
    return LandmarkConsensus(h, float(cons.get("thresh", 0.0)), int(cons.get("min_inliers", 0)), int(cons.get("seed", 0)) % 2 ** 64,
                             scores.ctypes.data), (scores,)


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(str(lib_path()))
        _lib.msckf_b200_last_error.restype = C.c_char_p
        _lib.msckf_b200_launch_count.restype = C.c_longlong
        _lib.msckf_b200_stream.restype = C.c_void_p
    return _lib


def check(rc, what):
    if rc < 0:
        raise RuntimeError(f"{what} failed rc={rc}: {(lib().msckf_b200_last_error() or b'').decode()}")
    return rc


class TrackBatch:
    """host-side flat SoA batch (keeps the numpy arrays alive)."""

    def __init__(self, obs_offset, obs, clone_index, dtype, p_f_G=None):
        self.dtype = np.dtype(dtype)
        self.off = np.ascontiguousarray(obs_offset, dtype=np.int32)
        self.obs = np.ascontiguousarray(obs, dtype=self.dtype)
        self.idx = np.ascontiguousarray(clone_index, dtype=np.int32)
        self.pfg = None if p_f_G is None else np.ascontiguousarray(p_f_G, dtype=self.dtype)
        self.c = Tracks(len(self.off) - 1, self.off.ctypes.data_as(C.POINTER(C.c_int)), self.obs.ctypes.data_as(C.c_void_p),
                        self.idx.ctypes.data_as(C.POINTER(C.c_int)), None if self.pfg is None else self.pfg.ctypes.data_as(C.c_void_p))

    @property
    def n_tracks(self):
        return len(self.off) - 1

    def h2d_bytes(self):
        return self.off.nbytes + self.obs.nbytes + self.idx.nbytes + (0 if self.pfg is None else self.pfg.nbytes)


def _report(n_tracks, dtype, full=True):
    """(Report, its per-track host arrays): accepted [n] and, with full, cm_ok, tri_ok, valid [n], gamma [n] and p_f_G [n, 3] in
    the filter's dtype"""
    k = max(n_tracks, 1)
    arr = {"accepted": np.zeros(k, np.int32)}
    if full:
        arr.update(cm_ok=np.zeros(k, np.int32), tri_ok=np.zeros(k, np.int32), valid=np.zeros(k, np.int32),
                   gamma=np.zeros(k, dtype), p_f_G=np.zeros((k, 3), dtype))
    rep = Report()
    for key in ("cm_ok", "tri_ok", "valid", "accepted"):
        if key in arr:
            setattr(rep, key, arr[key].ctypes.data_as(C.POINTER(C.c_int)))
    if full:
        rep.gamma, rep.p_f_G = arr["gamma"].ctypes.data, arr["p_f_G"].ctypes.data
    return rep, arr


def _result(rep, arr, n_tracks):
    """the report as a dict: m, rank and the per-track arrays (the flags and p_f_G of the modes that compute them)"""
    return dict({k: v[:n_tracks] for k, v in arr.items()}, m=rep.m, rank=rep.rank)


class Batch:
    """msckf_b200_batch: n engines whose updates run as ONE device batch (filter index in blockIdx.z, one CUDA graph, one
    packed copy each way).  While it lives the engines share its stream."""

    def __init__(self, engines):
        self.engines = list(engines)
        n = len(self.engines)
        hs = (C.c_void_p * n)(*[e.h for e in self.engines])
        self.h = C.c_void_p()
        check(lib().msckf_b200_batch_create(hs, C.c_int(n), C.byref(self.h)), "msckf_b200_batch_create")
        lib().msckf_b200_batch_launch_count.restype = C.c_longlong

    def close(self):
        if self.h:
            lib().msckf_b200_batch_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _tracks(self, batches):
        assert len(batches) == len(self.engines)
        return (Tracks * len(batches))(*[b.c for b in batches])

    def stage(self, mode, batches, threads=1):
        self._keep = batches
        check(lib().msckf_b200_batch_stage(self.h, C.c_int(mode), self._tracks(batches), C.c_int(threads)), "msckf_b200_batch_stage")

    def launch(self):
        check(lib().msckf_b200_batch_launch(self.h), "msckf_b200_batch_launch")

    def launch_timed(self):
        ms = C.c_float()
        check(lib().msckf_b200_batch_launch_timed(self.h, C.byref(ms)), "msckf_b200_batch_launch_timed")
        return ms.value

    def _reports(self, batches, full):
        st = [_report(b.n_tracks, e.dtype, full) for b, e in zip(batches, self.engines)]
        return (Report * len(st))(*[r for r, _ in st]), [a for _, a in st]

    def fetch(self, batches=None, full=False):
        """per engine m, rank, accepted and, with full, the other per-track results (see Engine.update)"""
        batches = batches or self._keep
        reps, arrs = self._reports(batches, full)
        check(lib().msckf_b200_batch_fetch(self.h, reps), "msckf_b200_batch_fetch")
        return [_result(r, a, b.n_tracks) for r, a, b in zip(reps, arrs, batches)]

    def update(self, mode, batches, threads=1, full=False):
        """host buffers in, reports out: packing + one H2D + kernels + one D2H (the batch's end-to-end call)."""
        reps, arrs = self._reports(batches, full)
        check(lib().msckf_b200_batch_update(self.h, C.c_int(mode), self._tracks(batches), reps, C.c_int(threads)), "msckf_b200_batch_update")
        return [_result(r, a, b.n_tracks) for r, a, b in zip(reps, arrs, batches)]

    def kernel_times(self):
        ms = (C.c_float * 32)()
        names = (C.c_char_p * 32)()
        n = check(lib().msckf_b200_batch_kernel_times(self.h, ms, names, C.c_int(32)), "msckf_b200_batch_kernel_times")
        return [(names[i].decode(), ms[i]) for i in range(n)]

    def launch_count(self):
        return int(lib().msckf_b200_batch_launch_count(self.h))

    def propagate_n(self, readings):
        """msckf_b200_batch_propagate_n: readings[i] = [k_i, 7] array (k_i may be 0) for engine i"""
        n = len(self.engines)
        assert len(readings) == n
        rs = [np.ascontiguousarray(r, dtype=e.dtype).reshape(-1, 7) for r, e in zip(readings, self.engines)]
        ptrs = (C.c_void_p * n)(*[r.ctypes.data if len(r) else None for r in rs])
        k = (C.c_int * n)(*[len(r) for r in rs])
        check(lib().msckf_b200_batch_propagate_n(self.h, ptrs, k), "msckf_b200_batch_propagate_n")

    def augment(self, which=None):
        """msckf_b200_batch_augment for the engines with which[i] (None: all)"""
        w = None if which is None else (C.c_int * len(self.engines))(*[int(bool(x)) for x in which])
        check(lib().msckf_b200_batch_augment(self.h, w), "msckf_b200_batch_augment")

    def prune(self, keeps):
        """msckf_b200_batch_prune: keeps[i] = ascending positions to keep, or None (engine i untouched)"""
        n = len(self.engines)
        ks = [None if k is None else np.ascontiguousarray(k, dtype=np.int32) for k in keeps]
        ptrs = (C.POINTER(C.c_int) * n)(*[None if k is None else k.ctypes.data_as(C.POINTER(C.c_int)) for k in ks])
        nk = (C.c_int * n)(*[-1 if k is None else len(k) for k in ks])
        check(lib().msckf_b200_batch_prune(self.h, ptrs, nk), "msckf_b200_batch_prune")

    def state(self):
        """msckf_b200_batch_get_state: [(imu [29], clone poses [M, 7])] per engine, with one synchronisation"""
        n = len(self.engines)
        out = [(np.zeros(29, dtype=e.dtype), np.zeros((e.num_clones(), 7), dtype=e.dtype)) for e in self.engines]
        imu = (C.c_void_p * n)(*[o[0].ctypes.data for o in out])
        poses = (C.c_void_p * n)(*[o[1].ctypes.data if o[1].size else None for o in out])
        check(lib().msckf_b200_batch_get_state(self.h, imu, poses), "msckf_b200_batch_get_state")
        return out

    def nees(self, truth_imus, truth_poses=None):
        """msckf_b200_batch_nees: NEES of every engine against its truth (truth_poses None, or per engine None / [M_i, 7]);
        a list of dicts (orientation, position, pose, imu, full, dim_full, first_bad_pivot)"""
        n = len(self.engines)
        tp = truth_poses if truth_poses is not None else [None] * n
        ts = [_truth(i, p) for i, p in zip(truth_imus, tp)]
        zeros = np.zeros(7)
        imu = (C.c_void_p * n)(*[t[0].ctypes.data for t in ts])
        poses = None if truth_poses is None else (C.c_void_p * n)(*[None if t[1] is None else (t[1].ctypes.data if t[1].size else zeros.ctypes.data) for t in ts])
        out = (NeesResult * n)()
        check(lib().msckf_b200_batch_nees(self.h, imu, poses, out), "msckf_b200_batch_nees")
        return [o.as_dict() for o in out]

    def aid_update(self, specs):
        """msckf_b200_batch_aid_update: specs[i] for engine i (see aid_struct; None leaves engine i alone); a list of result
        dicts (None for an engine left alone)"""
        n = len(self.engines)
        assert len(specs) == n
        st = [aid_struct(s) for s in specs]
        out = (AidResult * n)()
        check(lib().msckf_b200_batch_aid_update(self.h, (Aid * n)(*[a for a, _ in st]), out), "msckf_b200_batch_aid_update")
        return [None if s is None or s["model"] < 0 else o.as_dict() for s, o in zip(specs, out)]

    def aid_stack_update(self, stacks, chi2_max=0.0, fde=None, max_iter=None, tol=None):
        """msckf_b200_batch_aid_stack_update: stacks[i] = list of item dicts for engine i (see aid_items; None or [] leaves
        engine i alone); a list of result dicts (None for an engine left alone).  fde (see fde_struct):
        msckf_b200_batch_aid_stack_update_fde instead (chi2_max unused); each dict then has outcome, n_excluded and items.
        max_iter / tol (a number for every engine or one per engine; see Engine.aid_stack_update): the _iter forms, and each
        dict also has iterations, converged and step"""
        n = len(self.engines)
        assert len(stacks) == n
        st = [aid_items(s or []) for s in stacks]
        ptrs = (C.POINTER(AidItem) * n)(*[C.cast(a, C.POINTER(AidItem)) for a, _ in st])
        cnt = (C.c_int * n)(*[len(s or []) for s in stacks])
        it = None if max_iter is None and tol is None else aid_iter_structs(n, max_iter, tol)
        iout = (AidIterResult * n)()
        if fde is not None:
            f, out = fde_struct(fde), (AidFdeResult * n)()
            if it is None:
                check(lib().msckf_b200_batch_aid_stack_update_fde(self.h, ptrs, cnt, C.byref(f), out), "msckf_b200_batch_aid_stack_update_fde")
            else:
                check(lib().msckf_b200_batch_aid_stack_update_fde_iter(self.h, ptrs, cnt, C.byref(f), it, out, iout),
                      "msckf_b200_batch_aid_stack_update_fde_iter")
            res = [o.as_dict(len(s)) if s else None for s, o in zip(stacks, out)]
        else:
            out = (AidResult * n)()
            if it is None:
                check(lib().msckf_b200_batch_aid_stack_update(self.h, ptrs, cnt, C.c_double(chi2_max), out), "msckf_b200_batch_aid_stack_update")
            else:
                check(lib().msckf_b200_batch_aid_stack_update_iter(self.h, ptrs, cnt, C.c_double(chi2_max), it, out, iout),
                      "msckf_b200_batch_aid_stack_update_iter")
            res = [o.as_dict() if s else None for s, o in zip(stacks, out)]
        if it is not None:
            for r, o in zip(res, iout):
                if r is not None:
                    r.update(o.as_dict())
        return res

    def standstill_update(self, readings, cfg):
        """msckf_b200_batch_standstill_update: readings[i] = [k_i, 7] array (omega, a, dT) for engine i, or None / k_i = 0
        (engine i left alone); cfg as for standstill_struct.  A list of result dicts (the stack's nis, dx_norm, dof, applied,
        status, then scatter and outcome; None for an engine left alone)."""
        n = len(self.engines)
        assert len(readings) == n
        rs = [np.zeros((0, 7), dtype=e.dtype) if r is None else np.ascontiguousarray(r, dtype=e.dtype).reshape(-1, 7)
              for r, e in zip(readings, self.engines)]
        ptrs = (C.c_void_p * n)(*[r.ctypes.data if len(r) else None for r in rs])
        k = (C.c_int * n)(*[len(r) for r in rs])
        c, out = standstill_struct(cfg), (StandstillResult * n)()
        check(lib().msckf_b200_batch_standstill_update(self.h, ptrs, k, C.byref(c), out), "msckf_b200_batch_standstill_update")
        return [o.as_dict() if len(r) else None for r, o in zip(rs, out)]

    def landmark_update(self, specs, max_iter=None, tol=None, consensus=None):
        """msckf_b200_batch_landmark_update: specs[i] for engine i (see landmark_struct; None or no observations leaves engine
        i alone); max_iter / tol, when given, apply to every spec that does not set its own.  When a spec has Sigma_L (see
        landmark_map_struct) the call is msckf_b200_batch_map_landmark_update.  A list of result dicts with "gamma" and "flag"
        arrays (None for an engine left alone).  consensus (see consensus_struct; also a spec's own "consensus", which comes
        first): msckf_b200_batch_landmark_update_consensus, and each dict has a "consensus" dict with the hypotheses' scores."""
        n = len(self.engines)
        assert len(specs) == n
        extra = {k: v for k, v in (("max_iter", max_iter), ("tol", tol)) if v is not None}
        st = [landmark_struct(s if s is None else dict(extra, **s)) for s in specs]
        out = (LandmarkResult * n)()
        arr = (Landmarks * n)(*[a for a, _ in st])
        cs = [s.get("consensus", consensus) if s is not None else consensus for s in specs]
        if any(c is not None for c in cs):
            cons = [consensus_struct(c) for c in cs]
            cout = (LandmarkConsensusResult * n)()
            maps = [landmark_map_struct(s) for s in specs]
            check(lib().msckf_b200_batch_landmark_update_consensus(self.h, arr, (LandmarkMap * n)(*[m for m, _ in maps]),
                                                                   (LandmarkConsensus * n)(*[c for c, _ in cons]), out, cout),
                  "msckf_b200_batch_landmark_update_consensus")
            return [None if not k else dict(o.as_dict(), gamma=k[4], flag=k[5], consensus=co.as_dict(ck[0] if ck else None))
                    for (a, k), o, co, (c, ck) in zip(st, out, cout, cons)]
        if any(s is not None and s.get("Sigma_L") is not None for s in specs):
            maps = [landmark_map_struct(s) for s in specs]
            check(lib().msckf_b200_batch_map_landmark_update(self.h, arr, (LandmarkMap * n)(*[m for m, _ in maps]), out),
                  "msckf_b200_batch_map_landmark_update")
        else:
            check(lib().msckf_b200_batch_landmark_update(self.h, arr, out), "msckf_b200_batch_landmark_update")
        return [None if not k else dict(o.as_dict(), gamma=k[4], flag=k[5]) for (a, k), o in zip(st, out)]

    def jac_occupancy(self):
        """CTAs of k_jac resident per SM at the shape of the last launch (0 before the first)."""
        return int(lib().msckf_b200_batch_jac_occupancy(self.h))


def update_batch(engines, mode, batches, threads=8):
    """msckf_b200_update_batch: one update per engine (independent filters), host work on `threads` threads.
    Returns the per-engine (m, rank, accepted) reports."""
    n = len(engines)
    assert n == len(batches)
    hs = (C.c_void_p * n)(*[e.h for e in engines])
    trs = (Tracks * n)(*[b.c for b in batches])
    reps = (Report * n)()
    accs = []
    for i, b in enumerate(batches):
        acc = np.zeros(max(b.n_tracks, 1), dtype=np.int32)
        reps[i].accepted = acc.ctypes.data_as(C.POINTER(C.c_int))
        accs.append(acc)
    check(lib().msckf_b200_update_batch(hs, C.c_int(n), C.c_int(mode), trs, reps, C.c_int(int(threads))), "msckf_b200_update_batch")
    return [{"m": reps[i].m, "rank": reps[i].rank, "accepted": accs[i][:batches[i].n_tracks]} for i in range(n)]


class Engine:
    """owning wrapper of a msckf_b200_engine*; `borrowed` wraps a handle owned by somebody else."""

    def __init__(self, dtype=np.float32, device=0, max_clones=40, max_tracks=512, max_obs=512 * 30, borrowed=None):
        self.dtype = np.dtype(dtype)
        self.owned = borrowed is None
        if borrowed is not None:
            self.h = C.c_void_p(borrowed)
        else:
            cfg = Config(0 if self.dtype == np.float32 else 1, device, max_clones, max_tracks, max_obs)
            self.h = C.c_void_p()
            check(lib().msckf_b200_create(C.byref(cfg), C.byref(self.h)), "msckf_b200_create")

    def close(self):
        if self.owned and self.h:
            lib().msckf_b200_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def copy_state_from(self, other):
        check(lib().msckf_b200_copy_state(self.h, other.h), "msckf_b200_copy_state")

    def stage(self, mode, batch):
        check(lib().msckf_b200_stage(self.h, C.c_int(mode), C.byref(batch.c)), "msckf_b200_stage")

    def launch(self):
        check(lib().msckf_b200_launch(self.h), "msckf_b200_launch")

    def launch_timed(self):
        ms = C.c_float()
        check(lib().msckf_b200_launch_timed(self.h, C.byref(ms)), "msckf_b200_launch_timed")
        return ms.value

    def fetch(self, n_tracks=0):
        rep = Report()
        acc = np.zeros(max(n_tracks, 1), dtype=np.int32)
        rep.accepted = acc.ctypes.data_as(C.POINTER(C.c_int))
        check(lib().msckf_b200_fetch(self.h, C.byref(rep)), "msckf_b200_fetch")
        return {"m": rep.m, "rank": rep.rank, "accepted": acc[:n_tracks]}

    def synchronize(self):
        check(lib().msckf_b200_synchronize(self.h), "msckf_b200_synchronize")

    def propagate_n(self, readings):
        r = np.ascontiguousarray(readings, dtype=self.dtype).reshape(-1, 7)
        check(lib().msckf_b200_propagate_n(self.h, r.ctypes.data_as(C.c_void_p), C.c_int(len(r))), "msckf_b200_propagate_n")

    def augment(self):
        check(lib().msckf_b200_augment(self.h), "msckf_b200_augment")

    def prune(self, keep):
        k = np.ascontiguousarray(keep, dtype=np.int32)
        check(lib().msckf_b200_prune(self.h, k.ctypes.data_as(C.POINTER(C.c_int)), C.c_int(len(k))), "msckf_b200_prune")

    def update(self, mode, batch):
        """one update; the report as a dict: m, rank and the per-track cm_ok, tri_ok, valid, accepted, gamma, p_f_G"""
        rep, arr = _report(batch.n_tracks, self.dtype)
        check(lib().msckf_b200_update(self.h, C.c_int(mode), C.byref(batch.c), C.byref(rep)), "msckf_b200_update")
        return _result(rep, arr, batch.n_tracks)

    def rank_pivots(self):
        n = check(lib().msckf_b200_rank_pivots(self.h, None, C.c_int(0)), "msckf_b200_rank_pivots")
        out = np.zeros(n)
        check(lib().msckf_b200_rank_pivots(self.h, out.ctypes.data_as(C.POINTER(C.c_double)), C.c_int(n)), "msckf_b200_rank_pivots")
        return out

    def set_option(self, key, value):
        check(lib().msckf_b200_set_option(self.h, C.c_int(key), C.c_double(value)), "msckf_b200_set_option")

    # msckf_b200_stage_buffer: name -> (which, element type (None: the filter's dtype), trailing shape; "n" = 15 + 6M, "c" = 6M)
    STAGE_BUFFERS = {"T2": (0, np.float64, ("n",)), "R2": (1, np.float64, ("n",)), "r2": (2, np.float64, ()),
                     "Z": (3, np.float64, ("c",)), "Yq": (4, np.float64, ("c",)), "ur": (5, np.float64, ()),
                     "D1": (6, np.float64, (6, 6)), "D2": (7, np.float64, (6, 6)), "bb": (8, np.float64, (6,)),
                     "Xg": (9, None, (2, 6)), "rg": (10, None, (2,)), "Vg": (11, None, (3,)), "taug": (12, None, (3,)),
                     "accept": (13, np.int32, ()), "row_off": (14, np.int32, ())}

    def stage_buffer(self, name):
        """one buffer of the last update's compression stage (see STAGE_BUFFERS and include/msckf_b200.h): T2, R2 [n, n];
        r2 [n]; Z, Yq [3N, c]; ur [3N]; D1, D2 [M, 6, 6]; bb [M, 6]; Xg [O, 2, 6], rg [O, 2], Vg [2O, 3], taug [N, 3] in the
        filter's dtype; accept [N], row_off [N + 1]; None when there is no such update"""
        def count(which):
            return check(lib().msckf_b200_stage_buffer(self.h, C.c_int(which), None, C.c_int(0)), "msckf_b200_stage_buffer")
        which, dt, shape = self.STAGE_BUFFERS[name]
        n = count(which)
        if n == 0:
            return None
        out = np.zeros(n, dtype=self.dtype if dt is None else dt)
        check(lib().msckf_b200_stage_buffer(self.h, C.c_int(which), out.ctypes.data_as(C.c_void_p), C.c_int(n)), "msckf_b200_stage_buffer")
        M = count(6) // 36  # the window of that update
        return out.reshape((-1,) + tuple({"n": 15 + 6 * M, "c": 6 * M}.get(d, d) for d in shape))

    def kernel_times(self):
        ms = (C.c_float * 32)()
        names = (C.c_char_p * 32)()
        n = check(lib().msckf_b200_kernel_times(self.h, ms, names, C.c_int(32)), "msckf_b200_kernel_times")
        return [(names[i].decode(), ms[i]) for i in range(n)]

    def launch_count(self):
        return int(lib().msckf_b200_launch_count(self.h))

    def num_clones(self):
        return lib().msckf_b200_num_clones(self.h)

    def jac_group(self):
        """threads per track k_jac ran with at the last update launch (after any widening; 0 before the first)"""
        return int(lib().msckf_b200_jac_group(self.h))

    def state(self):
        """(imu [29]: p, v, b_g, b_a, g, q_IG, p_null, v_null, q_null; clone poses [M, 7]: p, q), dtype scalars"""
        imu = np.zeros(29, dtype=self.dtype)
        poses = np.zeros((self.num_clones(), 7), dtype=self.dtype)
        check(lib().msckf_b200_get_state(self.h, imu.ctypes.data_as(C.c_void_p), poses.ctypes.data_as(C.c_void_p)), "msckf_b200_get_state")
        return imu, poses

    def nees(self, truth_imu, truth_poses=None):
        """msckf_b200_nees against truth_imu (19) and, optionally, the window's truth poses [M, 7]"""
        imu, poses = _truth(truth_imu, truth_poses)
        zeros = np.zeros(7)
        p = None if poses is None else C.c_void_p(poses.ctypes.data if poses.size else zeros.ctypes.data)
        out = NeesResult()
        check(lib().msckf_b200_nees(self.h, C.c_void_p(imu.ctypes.data), p, C.byref(out)), "msckf_b200_nees")
        return out.as_dict()

    def aid_update(self, model, z, R, H=None, clone=0, chi2_max=0.0):
        """msckf_b200_aid_update: one aided measurement (see aid_struct); the result as a dict"""
        a, keep = aid_struct({"model": model, "z": z, "R": R, "H": H, "clone": clone, "chi2_max": chi2_max})
        out = AidResult()
        check(lib().msckf_b200_aid_update(self.h, C.byref(a), C.byref(out)), "msckf_b200_aid_update")
        return out.as_dict()

    def aid_stack_update(self, items, chi2_max=0.0, fde=None, max_iter=None, tol=None):
        """msckf_b200_aid_stack_update: one stacked update of items (see aid_items); the result as a dict.  fde (see
        fde_struct): msckf_b200_aid_stack_update_fde instead (chi2_max unused); the dict then has outcome, n_excluded and items.
        max_iter (0..16; 0 or 1: one linearisation) / tol (finite, >= 0; None: 0): the iterated update
        (msckf_b200_aid_stack_update_iter / _fde_iter); the dict then also has iterations, converged and step.  With neither
        given the call is the one above."""
        arr, keep = aid_items(items)
        it = None if max_iter is None and tol is None else aid_iter_structs(1, max_iter, tol)
        iout = AidIterResult()
        if fde is not None:
            f, out = fde_struct(fde), AidFdeResult()
            if it is None:
                check(lib().msckf_b200_aid_stack_update_fde(self.h, arr, C.c_int(len(items)), C.byref(f), C.byref(out)),
                      "msckf_b200_aid_stack_update_fde")
            else:
                check(lib().msckf_b200_aid_stack_update_fde_iter(self.h, arr, C.c_int(len(items)), C.byref(f), it, C.byref(out),
                                                                 C.byref(iout)), "msckf_b200_aid_stack_update_fde_iter")
            res = out.as_dict(len(items))
        else:
            out = AidResult()
            if it is None:
                check(lib().msckf_b200_aid_stack_update(self.h, arr, C.c_int(len(items)), C.c_double(chi2_max), C.byref(out)),
                      "msckf_b200_aid_stack_update")
            else:
                check(lib().msckf_b200_aid_stack_update_iter(self.h, arr, C.c_int(len(items)), C.c_double(chi2_max), it,
                                                             C.byref(out), C.byref(iout)), "msckf_b200_aid_stack_update_iter")
            res = out.as_dict()
        if it is not None:
            res.update(iout.as_dict())
        return res

    def standstill_update(self, readings, cfg):
        """msckf_b200_standstill_update: readings [k, 7] (omega, a, dT; rounded to the engine's dtype), cfg as for
        standstill_struct.  The result as a dict: the stack's nis, dx_norm, dof, applied, status, then scatter and outcome."""
        r = np.ascontiguousarray(readings, dtype=self.dtype).reshape(-1, 7)
        c, out = standstill_struct(cfg), StandstillResult()
        check(lib().msckf_b200_standstill_update(self.h, C.c_void_p(r.ctypes.data), C.c_int(len(r)), C.byref(c), C.byref(out)),
              "msckf_b200_standstill_update")
        return out.as_dict()

    def landmark_update(self, clone, z, p_L, R=None, chi2_obs=0.0, max_iter=0, tol=0.0, landmark=None, Sigma_L=None, consensus=None):
        """msckf_b200_landmark_update: observations of known landmarks p_L [n, 3] at z [n, 2] from window positions clone [n];
        max_iter >= 2 iterates the update (at most max_iter linearisations, converged at max |delta_{i+1} - delta_i| <= tol).
        landmark [n] with Sigma_L (see landmark_map_struct): msckf_b200_map_landmark_update, each landmark's map error
        marginalised over its observations.  consensus (see consensus_struct): msckf_b200_landmark_update_consensus, and the
        dict has a "consensus" dict (status, inliers, best, valid, refit, yaw, t, pivot, scores).
        The result as a dict with the per-observation "gamma" and "flag" arrays"""
        a, keep = landmark_struct({"clone": clone, "z": z, "p_L": p_L, "R": R, "chi2_obs": chi2_obs, "max_iter": max_iter, "tol": tol})
        out = LandmarkResult()
        if consensus is not None:
            m, mk = landmark_map_struct(None if Sigma_L is None else {"landmark": landmark, "Sigma_L": Sigma_L})
            c, ck = consensus_struct(consensus)
            cout = LandmarkConsensusResult()
            check(lib().msckf_b200_landmark_update_consensus(self.h, C.byref(a), C.byref(m), C.byref(c), C.byref(out), C.byref(cout)),
                  "msckf_b200_landmark_update_consensus")
            return dict(out.as_dict(), gamma=keep[4] if keep else np.zeros(0), flag=keep[5] if keep else np.zeros(0, np.int32),
                        consensus=cout.as_dict(ck[0] if ck else None))
        if Sigma_L is None:
            check(lib().msckf_b200_landmark_update(self.h, C.byref(a), C.byref(out)), "msckf_b200_landmark_update")
        else:
            m, mk = landmark_map_struct({"landmark": landmark, "Sigma_L": Sigma_L})
            check(lib().msckf_b200_map_landmark_update(self.h, C.byref(a), C.byref(m), C.byref(out)), "msckf_b200_map_landmark_update")
        return dict(out.as_dict(), gamma=keep[4] if keep else np.zeros(0), flag=keep[5] if keep else np.zeros(0, np.int32))

    def covariance(self):
        n = 15 + 6 * self.num_clones()
        out = np.zeros((n, n), dtype=self.dtype)
        check(lib().msckf_b200_get_covariance(self.h, out.ctypes.data_as(C.c_void_p)), "msckf_b200_get_covariance")
        return out

    def set_covariance(self, P):
        P = np.ascontiguousarray(P, dtype=self.dtype)
        check(lib().msckf_b200_set_covariance(self.h, P.ctypes.data_as(C.c_void_p)), "msckf_b200_set_covariance")

    def poison_covariance(self):
        """test hook: a NaN in the IMU block (exercises MSCKF_B200_ERR_NUMERIC)"""
        P = self.covariance()
        P[0, 0] = np.nan
        self.set_covariance(P)

    def delta_x(self):
        out = np.zeros(15 + 6 * self.num_clones())
        n = check(lib().msckf_b200_last_delta_x(self.h, out.ctypes.data_as(C.POINTER(C.c_double)), C.c_int(len(out))), "last_delta_x")
        return out[:n].copy()
