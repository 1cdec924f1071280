"""ctypes binding of the "C view of msckf_mono::MSCKF<_S>" (include/msckf_mono_c.h).

The same function set is exported by the H100 engine (libmsckf_b200.so, prefix
``msckf_mono_``) and -- for tests and the CPU baseline only -- by the oracle
(oracle/libmsckf_oracle.so, prefix ``msckf_oracle_``); this class is prefix-agnostic so the
parity tests drive both through identical calls.  All scalars cross the boundary as double.
"""
from __future__ import annotations

import ctypes as C
import numpy as np

_dp = C.POINTER(C.c_double)
_u64p = C.POINTER(C.c_uint64)
_ip = C.POINTER(C.c_int)


def _d(a):
    a = np.ascontiguousarray(a, dtype=np.float64)
    return a, a.ctypes.data_as(_dp)


def pack_camera(cam):
    return np.concatenate([[cam["c_u"], cam["c_v"], cam["f_u"], cam["f_v"], cam["b"]],
                           np.asarray(cam["q_CI"], float), np.asarray(cam["p_C_I"], float)])


def pack_noise(nz):
    return np.concatenate([[nz["u_var_prime"], nz["v_var_prime"]], np.asarray(nz["Q_imu"], float).ravel(),
                           np.asarray(nz["initial_imu_covar"], float).ravel()])


def pack_params(p):
    return np.array([p["max_gn_cost_norm"], p["min_rcond"], p["translation_threshold"],
                     p["redundancy_angle_thresh"], p["redundancy_distance_thresh"],
                     p["min_track_length"], p["max_track_length"], p["max_cam_states"]], dtype=float)


def pack_imu_state(s):
    return np.concatenate([np.asarray(s[k], float) for k in ("p_I_G", "v_I_G", "b_g", "b_a", "g", "q_IG")])


NEES_KEYS = ("orientation", "position", "pose", "imu", "full", "dim_full", "first_bad_pivot")


def _nees_dict(o):
    d = dict(zip(NEES_KEYS, (float(x) for x in o)))
    d["dim_full"], d["first_bad_pivot"] = int(o[5]), int(o[6])
    return d


def _truth(truth_imu, truth_poses):
    imu = np.ascontiguousarray(truth_imu, dtype=np.float64).ravel()
    assert imu.size == 19, imu.size
    poses = None if truth_poses is None else np.ascontiguousarray(truth_poses, dtype=np.float64).reshape(-1, 7)
    if poses is not None and poses.size == 0:
        poses = np.zeros((1, 7))  # (an empty window: a valid pointer with nothing to read)
    return imu, poses


def marginalize_batch(filters, threads=8):
    """marginalize() on independent filters through the C view's batched entry point: launch on all, collect on all, the
    per-filter host work spread over `threads` host threads (engine filters only)."""
    if not filters:
        return
    f0 = filters[0]
    arr = (C.c_void_p * len(filters))(*[f.h for f in filters])
    f0._chk(f0._f("marginalize_batch")(arr, C.c_int(len(filters)), C.c_int(int(threads))), "marginalize_batch")



def _tri6(Sigma):
    """covariances [L, 3, 3] or [L, 6] as contiguous lower triangles xx, yx, yy, zx, zy, zz [L, 6]"""
    S = np.asarray(Sigma, dtype=np.float64)
    if S.ndim == 3:
        S = S[:, [0, 1, 1, 2, 2, 2], [0, 0, 1, 0, 1, 2]]
    return np.ascontiguousarray(S.reshape(-1, 6))

class FilterBatch:
    """msckf_mono::MSCKFBatch<_S> through the C view: a persistent device batch over engine filters of one dtype."""

    def __init__(self, filters, threads=1):
        self.filters = list(filters)
        f0 = self.filters[0]
        self.lib = f0.lib
        arr = (C.c_void_p * len(self.filters))(*[f.h for f in self.filters])
        self.h = C.c_void_p()
        f0._chk(self.lib.msckf_mono_batch_create(arr, C.c_int(len(self.filters)), C.c_int(int(threads)), C.byref(self.h)), "batch_create")

    def _call(self, name, *args):
        self.filters[0]._chk(getattr(self.lib, "msckf_mono_batch_" + name)(self.h, *args), "batch_" + name)

    def propagate(self, i, omega, a, dT):
        """MSCKF::propagate of filter i (queued; the batch hands every filter's queue over in one call)"""
        m, pm = _d(self.filters[0]._round(np.concatenate([omega, a, [dT]])))  # (one scalar type per batch)
        self._call("propagate", C.c_int(int(i)), pm)

    def augmentState(self, state_ids, times):
        """MSCKF::augmentState of every filter: state_ids[i], times[i] for filter i"""
        assert len(state_ids) == len(times) == len(self.filters)
        ids = np.ascontiguousarray(state_ids, dtype=np.int32)
        t, pt = _d([float(f._round(x)) for f, x in zip(self.filters, times)])
        self._call("augment_state", ids.ctypes.data_as(_ip), pt)

    def marginalize(self):
        self._call("marginalize")

    def pruneRedundantStates(self):
        self._call("prune_redundant_states")

    def pruneEmptyStates(self):
        self._call("prune_empty_states")

    def finish(self):
        self._call("finish")

    def refreshState(self):
        """every filter's IMU state and clone poses with one synchronisation"""
        self._call("refresh_state")

    def nees(self, truth_imus, truth_poses=None):
        """MSCKFBatch::nees: every filter against its truth (19 doubles) and, per filter, its window's truth poses [M, 7]
        or None; one device call for the batch.  A list of dicts."""
        n = len(self.filters)
        tp = truth_poses if truth_poses is not None else [None] * n
        ts = [_truth(i, p) for i, p in zip(truth_imus, tp)]
        imu = (C.c_void_p * n)(*[t[0].ctypes.data for t in ts])
        poses = None if truth_poses is None else (C.c_void_p * n)(*[None if t[1] is None else t[1].ctypes.data for t in ts])
        out = np.zeros((n, 7))
        self._call("nees", imu, poses, out.ctypes.data_as(_dp))
        return [_nees_dict(o) for o in out]

    def aid_update(self, specs):
        """MSCKFBatch::aidedUpdate: specs[i] for filter i (a dict as for capi.aid_struct, or None: filter i left alone); one
        device call for the batch.  A list of result dicts (None for a filter left alone)."""
        from .capi import Aid, AidResult, aid_struct
        n = len(self.filters)
        assert len(specs) == n
        st = [aid_struct(s) for s in specs]
        out = (AidResult * n)()
        self._call("aid_update", (Aid * n)(*[a for a, _ in st]), out)
        return [None if s is None or s["model"] < 0 else o.as_dict() for s, o in zip(specs, out)]

    def aid_stack_update(self, stacks, chi2_max=0.0, fde=None, max_iter=None, tol=None):
        """MSCKFBatch::aidedUpdate(items): stacks[i] = list of item dicts for filter i (as for capi.aid_items; None or []:
        filter i left alone); one device call for the batch.  A list of result dicts (None for a filter left alone).  fde (as for
        capi.fde_struct): MSCKFBatch::aidedUpdate(items, fde) instead; each dict then has outcome, n_excluded and items.
        max_iter / tol (a number for every filter or one per filter, as for capi.Batch.aid_stack_update): the iterated forms
        (MSCKFBatch::aidedUpdate(items, chi2_max | fde, iter, iter_out)); each dict then also has iterations, converged, step."""
        from .capi import AidFdeResult, AidIterResult, AidResult, aid_items, aid_iter_structs, fde_struct
        n = len(self.filters)
        assert len(stacks) == n
        flat = [it for s in stacks for it in (s or [])]
        arr, keep = aid_items(flat)
        cnt = np.array([len(s or []) for s in stacks], dtype=np.int32)
        it = None if max_iter is None and tol is None else aid_iter_structs(n, max_iter, tol)
        iout = (AidIterResult * n)()
        if fde is not None:
            f, out = fde_struct(fde), (AidFdeResult * n)()
            if it is None:
                self._call("aid_stack_update_fde", cnt.ctypes.data_as(_ip), arr, C.byref(f), out)
            else:
                self._call("aid_stack_update_fde_iter", cnt.ctypes.data_as(_ip), arr, C.byref(f), it, out, iout)
            res = [o.as_dict(len(s)) if s else None for s, o in zip(stacks, out)]
        else:
            out = (AidResult * n)()
            if it is None:
                self._call("aid_stack_update", cnt.ctypes.data_as(_ip), arr, C.c_double(chi2_max), out)
            else:
                self._call("aid_stack_update_iter", cnt.ctypes.data_as(_ip), arr, C.c_double(chi2_max), it, out, iout)
            res = [o.as_dict() if s else None for s, o in zip(stacks, out)]
        if it is not None:
            for r, o in zip(res, iout):
                if r is not None:
                    r.update(o.as_dict())
        return res

    def standstill_update(self, readings, cfg):
        """MSCKFBatch::standstillUpdate: readings[i] = [k_i, 7] (omega, a, dT) for filter i, or None / k_i = 0 (filter i left
        alone); cfg as for capi.standstill_struct; one device call for the batch.  A list of result dicts (None for a filter
        left alone)."""
        from .capi import StandstillResult, standstill_struct
        n = len(self.filters)
        assert len(readings) == n
        rs = [np.zeros((0, 7)) if r is None else np.asarray(r, float).reshape(-1, 7) for r in readings]
        flat, pr = _d(np.concatenate(rs) if sum(len(r) for r in rs) else np.zeros(7))
        cnt = np.array([len(r) for r in rs], dtype=np.int32)
        c, out = standstill_struct(cfg), (StandstillResult * n)()
        self._call("standstill_update", cnt.ctypes.data_as(_ip), pr, C.byref(c), out)
        return [o.as_dict() if len(r) else None for r, o in zip(rs, out)]

    def map_update(self, obs, R=None, chi2_obs=0.0, max_iter=1, tol=1e-10):
        """MSCKFBatch::landmarkUpdate over mapObservation / mapLandmark: obs[i] = (state_ids [n], landmark [n], z [n, 2],
        p_L [L, 3], Sigma [L, 6] or [L, 3, 3]) for filter i, or None (left alone); one device call for the batch.  A list of
        result dicts with "gamma" and "flag" (None for a filter left alone)."""
        from .capi import LandmarkResult
        n = len(self.filters)
        assert len(obs) == n
        cnt = np.array([0 if o is None else len(o[0]) for o in obs], dtype=np.int32)
        nl = np.array([0 if o is None or not len(o[0]) else len(np.asarray(o[3]).reshape(-1, 3)) for o in obs], dtype=np.int32)
        parts = [o for o in obs if o is not None and len(o[0])]

        def cat(i, w, dt):
            return np.ascontiguousarray(np.concatenate([np.asarray(o[i], dt).reshape(-1, w) for o in parts]) if parts
                                        else np.zeros((1, w)), dtype=dt)
        ids, lm, z, p = cat(0, 1, np.int32), cat(1, 1, np.int32), cat(2, 2, float), cat(3, 3, float)
        S = np.ascontiguousarray(np.concatenate([_tri6(o[4]) for o in parts]) if parts else np.zeros((1, 6)))
        r3 = None if R is None else np.array([R[0][0], R[1][0], R[1][1]], dtype=np.float64)
        tot = max(int(cnt.sum()), 1)
        gamma, flag = np.zeros(tot), np.zeros(tot, dtype=np.int32)
        out = (LandmarkResult * n)()
        self._call("map_update", cnt.ctypes.data_as(_ip), ids.ctypes.data_as(_ip), lm.ctypes.data_as(_ip), z.ctypes.data_as(_dp),
                   nl.ctypes.data_as(_ip), p.ctypes.data_as(_dp), S.ctypes.data_as(_dp), None if r3 is None else r3.ctypes.data_as(_dp),
                   C.c_double(chi2_obs), C.c_int(int(max_iter)), C.c_double(tol), gamma.ctypes.data_as(_dp), flag.ctypes.data_as(_ip),
                   out)
        res, o0 = [], 0
        for i in range(n):
            c = int(cnt[i])
            res.append(None if c == 0 else dict(out[i].as_dict(), gamma=gamma[o0:o0 + c].copy(), flag=flag[o0:o0 + c].copy()))
            o0 += c
        return res

    def landmark_update(self, obs, R=None, chi2_obs=0.0, max_iter=1, tol=1e-10, consensus=None):
        """MSCKFBatch::landmarkUpdate: obs[i] = (state_ids [n], z [n, 2], p_L [n, 3]) for filter i, or None (filter i left
        alone); R None (each filter's pixel noise) or 2 x 2; one device call for the batch; max_iter >= 2: the iterated update
        (at most max_iter linearisations, converged at max |delta_{i+1} - delta_i| <= tol).  A list of result dicts with
        "gamma" and "flag" (None for a filter left alone).  consensus (a capi.consensus_struct dict, or one per filter):
        msckf_mono_batch_landmark_update_consensus, and each dict has a "consensus" dict."""
        from .capi import LandmarkResult
        n = len(self.filters)
        if consensus is not None:
            return self._landmark_consensus(obs, R, chi2_obs, max_iter, tol, consensus)
        assert len(obs) == n
        cnt = np.array([0 if o is None else len(o[0]) for o in obs], dtype=np.int32)
        parts = [o for o in obs if o is not None and len(o[0])]
        ids = np.ascontiguousarray(np.concatenate([np.asarray(o[0]) for o in parts]) if parts else np.zeros(1), dtype=np.int32)
        z = np.ascontiguousarray(np.concatenate([np.asarray(o[1], float).reshape(-1, 2) for o in parts]) if parts else np.zeros((1, 2)))
        p = np.ascontiguousarray(np.concatenate([np.asarray(o[2], float).reshape(-1, 3) for o in parts]) if parts else np.zeros((1, 3)))
        r3 = None if R is None else np.array([R[0][0], R[1][0], R[1][1]], dtype=np.float64)
        tot = max(int(cnt.sum()), 1)
        gamma, flag = np.zeros(tot), np.zeros(tot, dtype=np.int32)
        out = (LandmarkResult * n)()
        it = () if max_iter == 1 else (C.c_int(int(max_iter)), C.c_double(tol))
        self._call("landmark_update" + ("_iter" if it else ""), cnt.ctypes.data_as(_ip), ids.ctypes.data_as(_ip),
                   z.ctypes.data_as(_dp), p.ctypes.data_as(_dp), None if r3 is None else r3.ctypes.data_as(_dp),
                   C.c_double(chi2_obs), *it, gamma.ctypes.data_as(_dp), flag.ctypes.data_as(_ip), out)
        res, o0 = [], 0
        for i in range(n):
            c = int(cnt[i])
            res.append(None if c == 0 else dict(out[i].as_dict(), gamma=gamma[o0:o0 + c].copy(), flag=flag[o0:o0 + c].copy()))
            o0 += c
        return res

    def _landmark_consensus(self, obs, R, chi2_obs, max_iter, tol, consensus):
        from .capi import LandmarkConsensus, LandmarkConsensusResult, LandmarkResult, consensus_struct
        n = len(self.filters)
        assert len(obs) == n
        cl = list(consensus) if isinstance(consensus, (list, tuple)) else [consensus] * n
        cs = [consensus_struct(c) for c in cl]
        cnt = np.array([0 if o is None else len(o[0]) for o in obs], dtype=np.int32)
        parts = [o for o in obs if o is not None and len(o[0])]
        ids = np.ascontiguousarray(np.concatenate([np.asarray(o[0]) for o in parts]) if parts else np.zeros(1), dtype=np.int32)
        z = np.ascontiguousarray(np.concatenate([np.asarray(o[1], float).reshape(-1, 2) for o in parts]) if parts else np.zeros((1, 2)))
        p = np.ascontiguousarray(np.concatenate([np.asarray(o[2], float).reshape(-1, 3) for o in parts]) if parts else np.zeros((1, 3)))
        r3 = None if R is None else np.array([R[0][0], R[1][0], R[1][1]], dtype=np.float64)
        tot = max(int(cnt.sum()), 1)
        gamma, flag = np.zeros(tot), np.zeros(tot, dtype=np.int32)
        out, cout = (LandmarkResult * n)(), (LandmarkConsensusResult * n)()
        self._call("landmark_update_consensus", cnt.ctypes.data_as(_ip), ids.ctypes.data_as(_ip), z.ctypes.data_as(_dp),
                   p.ctypes.data_as(_dp), None if r3 is None else r3.ctypes.data_as(_dp), C.c_double(chi2_obs),
                   C.c_int(int(max_iter)), C.c_double(tol), (LandmarkConsensus * n)(*[c for c, _ in cs]),
                   gamma.ctypes.data_as(_dp), flag.ctypes.data_as(_ip), out, cout)
        res, o0 = [], 0
        for i in range(n):
            c = int(cnt[i])
            res.append(None if c == 0 else dict(out[i].as_dict(), gamma=gamma[o0:o0 + c].copy(), flag=flag[o0:o0 + c].copy(),
                                                consensus=cout[i].as_dict(cs[i][1][0] if cs[i][1] else None)))
            o0 += c
        return res

    def handle(self):
        fn = self.lib.msckf_mono_batch_handle
        fn.restype = C.c_void_p
        return fn(self.h)

    def close(self):
        if self.h:
            self.lib.msckf_mono_batch_destroy.argtypes = [C.c_void_p]
            self.lib.msckf_mono_batch_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class CFilter:
    """MSCKF<_S> surface over a C view.  dtype: np.float32 or np.float64."""

    def __init__(self, lib_path, prefix, dtype=np.float64, create_args=()):
        self.lib = C.CDLL(str(lib_path))
        self.prefix = prefix
        self.dtype = np.dtype(dtype)
        self.h = C.c_void_p()
        code = 0 if self.dtype == np.float32 else 1
        rc = self._f("create")(C.c_int(code), *create_args, C.byref(self.h))
        if rc != 0:
            raise RuntimeError(f"{prefix}create failed rc={rc}")

    def _f(self, name):
        return getattr(self.lib, self.prefix + name)

    def _chk(self, rc, what):
        if rc < 0:
            msg = ""
            try:
                fn = getattr(self.lib, self.prefix + "last_error")
                fn.restype = C.c_char_p
                msg = (fn() or b"").decode()
            except AttributeError:
                pass
            raise RuntimeError(f"{self.prefix}{what} failed rc={rc} {msg}")
        return rc

    def close(self):
        if self.h:
            self._f("destroy")(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _round(self, a):
        """inputs are rounded to the filter dtype first, so double(float(x)) is exact."""
        return np.asarray(a, dtype=self.dtype).astype(np.float64)

    # ---- MSCKF<_S> surface -------------------------------------------------------------
    def initialize(self, camera, noise, params, imu_state):
        a, pa = _d(self._round(pack_camera(camera)))
        b, pb = _d(self._round(pack_noise(noise)))
        c, pc = _d(pack_params({k: (self._round(v) if not isinstance(v, int) else v) for k, v in params.items()}))
        d, pd = _d(self._round(pack_imu_state(imu_state)))
        self._chk(self._f("initialize")(self.h, pa, pb, pc, pd), "initialize")

    def propagate(self, omega, a, dT):
        m, pm = _d(self._round(np.concatenate([omega, a, [dT]])))
        self._chk(self._f("propagate")(self.h, pm), "propagate")

    def augmentState(self, state_id, time):
        self._chk(self._f("augment_state")(self.h, C.c_int(int(state_id)), C.c_double(float(self._round(time)))), "augment_state")

    def _obs(self, z, ids):
        z = self._round(np.asarray(z, float).reshape(-1, 2))
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        assert len(ids) == len(z)
        return z, z.ctypes.data_as(_dp), ids, ids.ctypes.data_as(_u64p), C.c_int(len(ids))

    def update(self, z, ids):
        z, pz, ids, pi, n = self._obs(z, ids)
        self._chk(self._f("update")(self.h, pz, pi, n), "update")

    def addFeatures(self, z, ids):
        z, pz, ids, pi, n = self._obs(z, ids)
        self._chk(self._f("add_features")(self.h, pz, pi, n), "add_features")

    def marginalize(self):
        self._chk(self._f("marginalize")(self.h), "marginalize")

    def pruneRedundantStates(self):
        self._chk(self._f("prune_redundant_states")(self.h), "prune_redundant_states")

    def pruneEmptyStates(self):
        self._chk(self._f("prune_empty_states")(self.h), "prune_empty_states")

    def finish(self):
        self._chk(self._f("finish")(self.h), "finish")

    # ---- getters -----------------------------------------------------------------------
    def getNumCamStates(self):
        return self._chk(self._f("get_num_cam_states")(self.h), "get_num_cam_states")

    def getImuState(self):
        o = np.zeros(29)
        self._chk(self._f("get_imu_state")(self.h, o.ctypes.data_as(_dp)), "get_imu_state")
        return {"p_I_G": o[0:3], "v_I_G": o[3:6], "b_g": o[6:9], "b_a": o[9:12], "g": o[12:15], "q_IG": o[15:19],
                "p_I_G_null": o[19:22], "v_I_G_null": o[22:25], "q_IG_null": o[25:29]}

    def getCamStates(self):
        M = self.getNumCamStates()
        poses = np.zeros((max(M, 1), 7))
        ids = np.zeros((max(M, 1), 2), dtype=np.int32)
        times = np.zeros(max(M, 1))
        self._chk(self._f("get_cam_states")(self.h, poses.ctypes.data_as(_dp), ids.ctypes.data_as(_ip),
                                          times.ctypes.data_as(_dp)), "get_cam_states")
        return {"p_C_G": poses[:M, 0:3], "q_CG": poses[:M, 3:7], "state_id": ids[:M, 0],
                "last_correlated_id": ids[:M, 1], "time": times[:M]}

    def getCamTrackedIds(self, cam):
        cap = 4096
        out = np.zeros(cap, dtype=np.uint64)
        n = self._chk(self._f("get_cam_tracked_ids")(self.h, C.c_int(cam), out.ctypes.data_as(_u64p), C.c_int(cap)), "get_cam_tracked_ids")
        return out[:n].copy()

    def getCovariance(self):
        n = 15 + 6 * self.getNumCamStates()
        out = np.zeros((n, n))
        n2 = self._chk(self._f("get_covariance")(self.h, out.ctypes.data_as(_dp)), "get_covariance")
        assert n2 == n, (n2, n)
        return out

    def getMap(self):
        cap = 8192
        out = np.zeros((cap, 3))
        n = self._chk(self._f("get_map")(self.h, out.ctypes.data_as(_dp), C.c_int(cap)), "get_map")
        return out[:n].copy()

    def getPrunedStates(self):
        cap = 65536
        poses = np.zeros((cap, 7))
        ids = np.zeros((cap, 2), dtype=np.int32)
        n = self._chk(self._f("get_pruned_states")(self.h, poses.ctypes.data_as(_dp), ids.ctypes.data_as(_ip), C.c_int(cap)), "get_pruned_states")
        return {"p_C_G": poses[:n, :3].copy(), "q_CG": poses[:n, 3:].copy(), "state_id": ids[:n, 0].copy()}

    def getTrackedFeatureIds(self):
        cap = 65536
        out = np.zeros(cap, dtype=np.uint64)
        n = self._chk(self._f("get_tracked_feature_ids")(self.h, out.ctypes.data_as(_u64p), C.c_int(cap)), "get_tracked_feature_ids")
        return out[:n].copy()

    def nees(self, truth_imu, truth_poses=None):
        """MSCKF::nees against truth_imu (19 doubles: p, v, b_g, b_a, g, q_IG xyzw) and, optionally, the window's truth
        poses [M, 7] (p_C_G, q_CG xyzw): dict of orientation, position, pose, imu, full NEES, dim_full, first_bad_pivot"""
        imu, poses = _truth(truth_imu, truth_poses)
        out = np.zeros(7)
        self._chk(self._f("nees")(self.h, imu.ctypes.data_as(_dp), None if poses is None else poses.ctypes.data_as(_dp),
                                  out.ctypes.data_as(_dp)), "nees")
        return _nees_dict(out)

    def aid_update(self, model, z, R, H=None, clone=0, chi2_max=0.0):
        """MSCKF::aidedUpdate (include/msckf_b200.h: msckf_b200_aid_update): model, z (LINEAR: the residual), R [m, m],
        H [m, 15 + 6M] (LINEAR), clone (CLONE_POSE), chi2_max (> 0: NIS gate).  A dict nis, dx_norm, dof, applied, status."""
        from .capi import AidResult, aid_struct
        a, keep = aid_struct({"model": model, "z": z, "R": R, "H": H, "clone": clone, "chi2_max": chi2_max})
        out = AidResult()
        self._chk(self._f("aid_update")(self.h, C.byref(a), C.byref(out)), "aid_update")
        return out.as_dict()

    def aid_stack_update(self, items, chi2_max=0.0, fde=None, max_iter=None, tol=None):
        """MSCKF::aidedUpdate(items) (include/msckf_b200.h: msckf_b200_aid_stack_update): items as for capi.aid_items, one
        chi2_max for the stack.  A dict nis, dx_norm, dof, applied, status.  fde (as for capi.fde_struct):
        MSCKF::aidedUpdate(items, fde) (msckf_b200_aid_stack_update_fde) instead; the dict then has outcome, n_excluded, items.
        max_iter / tol (as for capi.Engine.aid_stack_update): MSCKF::aidedUpdate(items, chi2_max | fde, iter, iter_out)
        (msckf_b200_aid_stack_update_iter / _fde_iter); the dict then also has iterations, converged and step."""
        from .capi import AidFdeResult, AidIterResult, AidResult, aid_items, aid_iter_structs, fde_struct
        arr, keep = aid_items(items)
        it = None if max_iter is None and tol is None else aid_iter_structs(1, max_iter, tol)
        iout = AidIterResult()
        if fde is not None:
            f, out = fde_struct(fde), AidFdeResult()
            if it is None:
                self._chk(self._f("aid_stack_update_fde")(self.h, arr, C.c_int(len(items)), C.byref(f), C.byref(out)), "aid_stack_update_fde")
            else:
                self._chk(self._f("aid_stack_update_fde_iter")(self.h, arr, C.c_int(len(items)), C.byref(f), it, C.byref(out), C.byref(iout)),
                          "aid_stack_update_fde_iter")
            res = out.as_dict(len(items))
        else:
            out = AidResult()
            if it is None:
                self._chk(self._f("aid_stack_update")(self.h, arr, C.c_int(len(items)), C.c_double(chi2_max), C.byref(out)), "aid_stack_update")
            else:
                self._chk(self._f("aid_stack_update_iter")(self.h, arr, C.c_int(len(items)), C.c_double(chi2_max), it, C.byref(out),
                                                            C.byref(iout)), "aid_stack_update_iter")
            res = out.as_dict()
        if it is not None:
            res.update(iout.as_dict())
        return res

    def standstill_update(self, readings, cfg):
        """MSCKF::standstillUpdate (include/msckf_b200.h: msckf_b200_standstill_update): readings [k, 7] (omega, a, dT), cfg
        as for capi.standstill_struct.  A dict: the stack's nis, dx_norm, dof, applied, status, then scatter and outcome."""
        from .capi import StandstillResult, standstill_struct
        r, pr = _d(np.asarray(readings, float).reshape(-1, 7))
        c, out = standstill_struct(cfg), StandstillResult()
        self._chk(self._f("standstill_update")(self.h, pr, C.c_int(len(r)), C.byref(c), C.byref(out)), "standstill_update")
        return out.as_dict()

    def body_velocity_update(self, v_I, R, mask=7, chi2_max=0.0):
        """MSCKF::bodyVelocityUpdate: the IMU's velocity v_I in its own frame, rows selected by mask (bits 0..2), R over them"""
        from .capi import AidResult
        v, pv = _d(np.asarray(v_I, float).ravel())
        Rm, pR = _d(np.asarray(R, float))
        out = AidResult()
        self._chk(self._f("body_velocity_update")(self.h, pv, C.c_int(int(mask)), pR, C.c_double(chi2_max), C.byref(out)),
                  "body_velocity_update")
        return out.as_dict()

    def relative_pose_update(self, state_id_a, state_id_b, p, q, R, chi2_max=0.0):
        """MSCKF::relativePoseUpdate: the pose (p, q xyzw) of image state_id_b relative to image state_id_a, R 6 x 6"""
        from .capi import AidResult
        pa, pp = _d(np.asarray(p, float).ravel())
        qa, pq = _d(np.asarray(q, float).ravel())
        Rm, pR = _d(np.asarray(R, float))
        out = AidResult()
        self._chk(self._f("relative_pose_update")(self.h, C.c_int(int(state_id_a)), C.c_int(int(state_id_b)), pp, pq, pR,
                                                  C.c_double(chi2_max), C.byref(out)), "relative_pose_update")
        return out.as_dict()

    def map_update(self, state_ids, landmark, z, p_L, Sigma, R=None, chi2_obs=0.0, max_iter=1, tol=1e-10):
        """MSCKF::landmarkUpdate over mapObservation / mapLandmark (msckf_b200_map_landmark_update): observations z [n, 2] from
        the images state_ids [n] of the landmarks landmark [n] (indices into p_L [L, 3] and Sigma [L, 6] lower triangles or
        [L, 3, 3]); each landmark's map error is marginalised over its observations.  The result dict of landmark_update."""
        from .capi import LandmarkResult
        ids = np.ascontiguousarray(state_ids, dtype=np.int32).ravel()
        lm = np.ascontiguousarray(landmark, dtype=np.int32).ravel()
        n = len(ids)
        z, pz = _d(np.asarray(z, float).reshape(-1, 2) if n else np.zeros((1, 2)))
        p, pp = _d(np.asarray(p_L, float).reshape(-1, 3))
        S, ps = _d(_tri6(Sigma))
        r3 = None if R is None else np.array([R[0][0], R[1][0], R[1][1]], dtype=np.float64)
        gamma, flag = np.zeros(max(n, 1)), np.zeros(max(n, 1), dtype=np.int32)
        out = LandmarkResult()
        self._chk(self._f("map_update")(self.h, C.c_int(n), ids.ctypes.data_as(_ip), lm.ctypes.data_as(_ip), pz, C.c_int(len(p)), pp,
                                        ps, None if r3 is None else r3.ctypes.data_as(_dp), C.c_double(chi2_obs),
                                        C.c_int(int(max_iter)), C.c_double(tol), gamma.ctypes.data_as(_dp), flag.ctypes.data_as(_ip),
                                        C.byref(out)), "map_update")
        return dict(out.as_dict(), gamma=gamma[:n].copy(), flag=flag[:n].copy())

    def landmark_update(self, state_ids, z, p_L, R=None, chi2_obs=0.0, max_iter=1, tol=1e-10, consensus=None):
        """MSCKF::landmarkUpdate (include/msckf_b200.h: msckf_b200_landmark_update): observations of known landmarks p_L [n, 3]
        at z [n, 2] from the images state_ids [n]; R None (the filter's pixel noise) or 2 x 2; chi2_obs > 0: per-observation
        gate; max_iter >= 2: the iterated update.  A dict nis, dx_norm, dof, rows, used, applied, status, iterations,
        converged, step, gamma [n], flag [n].  consensus (a capi.consensus_struct dict): msckf_mono_landmark_update_consensus,
        and the dict has a "consensus" dict."""
        from .capi import LandmarkResult
        if consensus is not None:
            from .capi import LandmarkConsensusResult, consensus_struct
            ids = np.ascontiguousarray(state_ids, dtype=np.int32).ravel()
            n = len(ids)
            z, pz = _d(np.asarray(z, float).reshape(-1, 2) if n else np.zeros((1, 2)))
            p, pp = _d(np.asarray(p_L, float).reshape(-1, 3) if n else np.zeros((1, 3)))
            r3 = None if R is None else np.array([R[0][0], R[1][0], R[1][1]], dtype=np.float64)
            gamma, flag = np.zeros(max(n, 1)), np.zeros(max(n, 1), dtype=np.int32)
            c, ck = consensus_struct(consensus)
            out, cout = LandmarkResult(), LandmarkConsensusResult()
            self._chk(self._f("landmark_update_consensus")(self.h, C.c_int(n), ids.ctypes.data_as(_ip), pz, pp,
                                                           None if r3 is None else r3.ctypes.data_as(_dp), C.c_double(chi2_obs),
                                                           C.c_int(int(max_iter)), C.c_double(tol), C.byref(c),
                                                           gamma.ctypes.data_as(_dp), flag.ctypes.data_as(_ip), C.byref(out),
                                                           C.byref(cout)), "landmark_update_consensus")
            return dict(out.as_dict(), gamma=gamma[:n].copy(), flag=flag[:n].copy(), consensus=cout.as_dict(ck[0] if ck else None))
        ids = np.ascontiguousarray(state_ids, dtype=np.int32).ravel()
        n = len(ids)
        z, pz = _d(np.asarray(z, float).reshape(-1, 2) if n else np.zeros((1, 2)))
        p, pp = _d(np.asarray(p_L, float).reshape(-1, 3) if n else np.zeros((1, 3)))
        r3 = None if R is None else np.array([R[0][0], R[1][0], R[1][1]], dtype=np.float64)
        gamma, flag = np.zeros(max(n, 1)), np.zeros(max(n, 1), dtype=np.int32)
        out = LandmarkResult()
        it = () if max_iter == 1 else (C.c_int(int(max_iter)), C.c_double(tol))
        name = "landmark_update" + ("_iter" if it else "")
        self._chk(self._f(name)(self.h, C.c_int(n), ids.ctypes.data_as(_ip), pz, pp,
                                None if r3 is None else r3.ctypes.data_as(_dp), C.c_double(chi2_obs), *it,
                                gamma.ctypes.data_as(_dp), flag.ctypes.data_as(_ip), C.byref(out)), name)
        return dict(out.as_dict(), gamma=gamma[:n].copy(), flag=flag[:n].copy())

    # ---- test hooks --------------------------------------------------------------------
    def lastReport(self):
        cap = 8192
        flags = np.zeros((cap, 4), dtype=np.int32)
        gamma = np.zeros(cap)
        pfg = np.zeros((cap, 3))
        n = self._chk(self._f("last_report")(self.h, flags.ctypes.data_as(_ip), gamma.ctypes.data_as(_dp),
                                           pfg.ctypes.data_as(_dp), C.c_int(cap)), "last_report")
        return {"cm_passed": flags[:n, 0].copy(), "valid": flags[:n, 1].copy(), "accepted": flags[:n, 2].copy(),
                "rows": flags[:n, 3].copy(), "gamma": gamma[:n].copy(), "p_f_G": pfg[:n].copy()}

    def counters(self):
        out = (C.c_long * 8)()
        self._chk(self._f("get_counters")(self.h, out), "get_counters")
        return {"num_residualized": out[0], "pfg_shifted": out[1], "pfg_oob": out[2], "n_updates": out[3],
                "rows_kept": out[4], "m": out[5]}

    def setOption(self, key, value):
        self._chk(self._f("set_option")(self.h, C.c_int(key), C.c_double(value)), "set_option")

    def lastDeltaX(self):
        cap = 15 + 6 * 512
        out = np.zeros(cap)
        n = self._chk(self._f("last_delta_x")(self.h, out.ctypes.data_as(_dp), C.c_int(cap)), "last_delta_x")
        return out[:n].copy()

    def packQueued(self):
        """the batch queued by update()/finish() in the engine's flat SoA form (engine view only)."""
        cap_t, cap_o = 8192, 8192 * 64
        off = np.zeros(cap_t + 1, dtype=np.int32)
        obs = np.zeros(2 * cap_o)
        idx = np.zeros(cap_o, dtype=np.int32)
        n = self._chk(self._f("pack_queued")(self.h, off.ctypes.data_as(_ip), obs.ctypes.data_as(_dp), idx.ctypes.data_as(_ip),
                                            C.c_int(cap_t), C.c_int(cap_o)), "pack_queued")
        tot = int(off[n])
        return off[:n + 1].copy(), obs[:2 * tot].copy(), idx[:tot].copy()

    def engineHandle(self):
        fn = self._f("engine")
        fn.restype = C.c_void_p
        return fn(self.h)

    def marginalizeLaunch(self):
        self._chk(self._f("marginalize_launch")(self.h), "marginalize_launch")

    def marginalizeCollect(self):
        self._chk(self._f("marginalize_collect")(self.h), "marginalize_collect")

    def queuedTracks(self):
        cap = 8192
        ids = np.zeros(cap, dtype=np.uint64)
        nobs = np.zeros(cap, dtype=np.int32)
        n = self._chk(self._f("queued_tracks")(self.h, ids.ctypes.data_as(_u64p), nobs.ctypes.data_as(_ip), C.c_int(cap)), "queued_tracks")
        return ids[:n].copy(), nobs[:n].copy()
