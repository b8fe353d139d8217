"""Thin Python binding of the C-ABI (include/okvis_b200.h) -- the same calls a C++ host (the OKVIS
Estimator/Frontend shims, see INTEGRATION.md) makes.  No numerics live here."""
import ctypes as C

import numpy as np

from . import abi

_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = abi.load_library()
    return _lib


class OkbError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("okb error %d: %s" % (code, msg))
        self.code = code


def marg_job_fingerprint(job):
    """okb_marg_job_fingerprint: the hash landmark-sharded ranks compare (dense part of the job, not its landmarks)."""
    out = C.c_uint64(0)
    rc = lib().okb_marg_job_fingerprint(C.byref(job), C.byref(out))
    if rc != 0:
        raise OkbError(rc, "malformed job")
    return out.value


def _p(a):
    return C.c_void_p(a.ctypes.data) if a is not None else None


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


class Context:
    """okb_ctx: device memory for `max_windows` resident keyframe windows + the frontend buffers."""

    def __init__(self, device=0, max_windows=1):
        self._h = C.c_void_p()
        rc = lib().okb_ctx_create(int(device), int(max_windows), C.byref(self._h))
        if rc != 0:
            raise OkbError(rc, lib().okb_last_error(None).decode())
        self.max_windows = max_windows
        self._windows = {}

    def close(self):
        if self._h:
            lib().okb_ctx_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise OkbError(rc, lib().okb_last_error(self._h).decode())

    @property
    def kernel_launches(self):
        return int(lib().okb_kernel_launches(self._h))

    @property
    def stream(self):
        return lib().okb_stream(self._h)

    def profile_enable(self, on=True):
        self._check(lib().okb_profile_enable(self._h, int(on)))

    def set_solve_groups(self, n=0):
        """okb_set_solve_groups: window groups of later optimize calls, 0 = automatic, 1..4 forced."""
        self._check(lib().okb_set_solve_groups(self._h, int(n)))

    def profile_read(self):
        out = np.zeros(6)
        self._check(lib().okb_profile_read(self._h, _p(out)))
        return dict(landmarks_ms=out[0], landmarks_launches=int(out[1]), solve_ms=out[2], solve_launches=int(out[3]),
                    quality_ms=out[4], quality_launches=int(out[5]))

    # ---------------------------------------------------------------- landmark-sharded window (multi-GPU)
    def shard_export(self, rank, world, max_frames=32, max_landmarks=0):
        """okb_shard_export: allocates this rank's mailbox; returns the 64-byte IPC handle (numpy uint8).  max_landmarks > 0
        also reserves the landmark replica of the frontend calls for that many global landmark slots."""
        h = np.zeros(64, np.uint8)
        self._check(lib().okb_shard_reserve_landmarks(self._h, int(max_landmarks)))
        self._check(lib().okb_shard_export(self._h, int(rank), int(world), int(max_frames), _p(h)))
        return h

    def shard_connect(self, handles):
        h = np.ascontiguousarray(handles, dtype=np.uint8)
        self._check(lib().okb_shard_connect(self._h, _p(h)))

    @staticmethod
    def shard_connect_local(ctxs, max_frames=32, max_landmarks=0):
        for c in ctxs:
            c._check(lib().okb_shard_reserve_landmarks(c._h, int(max_landmarks)))
        arr = (C.c_void_p * len(ctxs))(*[c._h for c in ctxs])
        rc = lib().okb_shard_connect_local(arr, len(ctxs), int(max_frames))
        if rc != 0:
            raise OkbError(rc, "; ".join(lib().okb_last_error(c._h).decode() for c in ctxs))

    @staticmethod
    def shard_mailbox_layout(world, max_frames, max_landmarks):
        """okb_shard_mailbox_layout: (landmark replica offset, replica bytes, mailbox bytes) of one window slot."""
        out = np.zeros(3, np.uint64)
        rc = lib().okb_shard_mailbox_layout(int(world), int(max_frames), int(max_landmarks), _p(out))
        if rc != 0:
            raise OkbError(rc, "okb_shard_mailbox_layout: invalid arguments")
        return tuple(int(x) for x in out)

    def shard_stats(self, win=0):
        out = np.zeros(4)
        self._check(lib().okb_shard_stats(self._h, int(win), _p(out)))
        return dict(rounds=int(out[0]), wait_us=float(out[1]), fault=int(out[2]), epoch=int(out[3]))

    # ---------------------------------------------------------------- estimator path
    def upload(self, win, window):
        d = window.desc()
        self._check(lib().okb_window_upload(self._h, int(win), C.byref(d)))
        self._windows[win] = window

    # ---- resident window: incremental graph updates (no device work until commit / optimize / download)
    def reserve(self, win, max_frames, max_landmarks, max_observations, max_imu_samples, max_marg_dim=0):
        self._check(lib().okb_window_reserve(self._h, int(win), int(max_frames), int(max_landmarks), int(max_observations),
                                             int(max_imu_samples), int(max_marg_dim)))

    def add_frame(self, win, pose, speed_bias=None, term=None, samples=None):
        pose = _f64(pose)
        sb = _f64(speed_bias) if speed_bias is not None else None
        t = np.ascontiguousarray(term) if term is not None else None
        smp = np.ascontiguousarray(samples) if samples is not None else None
        self._check(lib().okb_window_add_frame(self._h, int(win), _p(pose), _p(sb), _p(t), _p(smp), 0 if smp is None else len(smp)))

    def remove_frame(self, win, pose_idx, sb_idx=None):
        self._check(lib().okb_window_remove_frame(self._h, int(win), C.c_uint32(int(pose_idx)),
                                                  C.c_uint32(0xffffffff if sb_idx is None else int(sb_idx))))

    def set_landmarks(self, win, idx, xyzw):
        idx = np.ascontiguousarray(idx, dtype=np.uint32)
        x = _f64(xyzw)
        self._check(lib().okb_window_set_landmarks(self._h, int(win), len(idx), _p(idx), _p(x)))

    def remove_landmarks(self, win, idx):
        idx = np.ascontiguousarray(idx, dtype=np.uint32)
        self._check(lib().okb_window_remove_landmarks(self._h, int(win), len(idx), _p(idx)))

    def add_observations(self, win, obs):
        obs = np.ascontiguousarray(obs, dtype=abi.observation_dtype)
        self._check(lib().okb_window_add_observations(self._h, int(win), len(obs), _p(obs)))

    def remove_observations(self, win, keys):
        k = np.zeros((len(keys), 4), np.uint32)
        k[:, :3] = np.asarray(keys, dtype=np.uint32).reshape(-1, 3)
        self._check(lib().okb_window_remove_observations(self._h, int(win), len(k), _p(k)))

    def set_states(self, win, pose_idx=(), poses=None, sb_idx=(), speed_bias=None):
        pi = np.ascontiguousarray(pose_idx, dtype=np.uint32)
        si = np.ascontiguousarray(sb_idx, dtype=np.uint32)
        self._check(lib().okb_window_set_states(self._h, int(win), len(pi), _p(pi) if len(pi) else None,
                                                _p(_f64(poses)) if len(pi) else None, len(si), _p(si) if len(si) else None,
                                                _p(_f64(speed_bias)) if len(si) else None))

    def set_priors(self, win, pose_priors, sb_priors, marg=None):
        pp = np.ascontiguousarray(pose_priors, dtype=abi.pose_prior_dtype)
        sp = np.ascontiguousarray(sb_priors, dtype=abi.sb_prior_dtype)
        m = None
        if marg is not None:
            m = abi.MargPrior()
            m.n, m.n_blocks = int(marg["J"].shape[0]), len(marg["block_kind"])
            m.block_kind = marg["block_kind"].ctypes.data_as(C.POINTER(C.c_int32))
            m.block_idx = marg["block_idx"].ctypes.data_as(C.POINTER(C.c_uint32))
            m.x0, m.J, m.e0 = abi.dptr(marg["x0"]), abi.dptr(marg["J"]), abi.dptr(marg["e0"])
        self._check(lib().okb_window_set_priors(self._h, int(win), len(pp), _p(pp) if len(pp) else None, len(sp),
                                                _p(sp) if len(sp) else None, C.byref(m) if m is not None else None))

    def remove_speed_bias(self, win, sb_idx):
        self._check(lib().okb_window_remove_speed_bias(self._h, int(win), C.c_uint32(int(sb_idx))))

    def marginalize(self, win, job):
        """okb_window_marginalize; job from abi.make_marg_job."""
        self._check(lib().okb_window_marginalize(self._h, int(win), C.byref(job)))

    def marginalize_batch(self, win_first, jobs):
        """okb_window_marginalize_batch: jobs[i] (from abi.make_marg_job, or None to leave the slot alone) runs on slot
        win_first + i."""
        arr = (C.POINTER(abi.MargJob) * max(len(jobs), 1))()
        for i, j in enumerate(jobs):
            if j is not None:
                arr[i] = C.pointer(j)
        self._check(lib().okb_window_marginalize_batch(self._h, int(win_first), len(jobs), arr))

    def download_marg(self, win):
        n, nb = C.c_int32(0), C.c_int32(0)
        kind, idx = np.zeros(64, np.int32), np.zeros(64, np.uint32)
        x0, J, e0, H, b0 = np.zeros(9 * 64), np.zeros(160 * 160), np.zeros(160), np.zeros(160 * 160), np.zeros(160)
        st = np.zeros(4, np.int32)
        self._check(lib().okb_window_download_marg(self._h, int(win), C.byref(n), C.byref(nb), _p(kind), _p(idx), _p(x0), _p(J),
                                                   _p(e0), _p(H), _p(b0), _p(st)))
        n, nb = n.value, nb.value
        kind, idx = kind[:nb].copy(), idx[:nb].copy()
        xdim = int(sum(9 if k == abi.BLOCK_SPEED_BIAS else 7 for k in kind))
        return dict(n=n, block_kind=kind, block_idx=idx, x0=x0[:xdim].copy(), J=J[:n * n].reshape(n, n).copy(), e0=e0[:n].copy(),
                    H=H[:n * n].reshape(n, n).copy(), b0=b0[:n].copy(), status=st.copy())

    def commit(self, first=0, count=1):
        self._check(lib().okb_window_commit(self._h, int(first), int(count)))

    def prepare_readd_newest(self, win, w):
        """Pre-marshalled arguments of the streaming pattern `drop the newest frame, add it again with its IMU term and
        observations` (what a VIO host does once per camera frame: Estimator::addStates + addObservation of that frame,
        okvis_ceres/src/Estimator.cpp:110-343, implementation/Estimator.hpp:43-90) for slot `win` holding window `w`."""
        K = len(w.poses)
        t = w.imu_terms[K - 2:K - 1].copy()
        lo, n = int(t["sample_offset"][0]), int(t["sample_count"][0])
        t["sample_offset"] = 0
        smp = np.ascontiguousarray(w.imu_samples[lo:lo + n])
        obs = np.ascontiguousarray(w.obs[w.obs["pose_idx"] == K - 1])
        pose, sb = _f64(w.poses[K - 1]).copy(), _f64(w.speed_bias[K - 1]).copy()
        keep = (pose, sb, t, smp, obs)
        return (C.c_int(int(win)), C.c_uint32(K - 1), _p(pose), _p(sb), _p(t), _p(smp), C.c_int(n), C.c_int(len(obs)), _p(obs), keep)

    def readd_newest(self, prepared):
        """Issues remove_frame / add_frame / add_observations for every prepared slot (host-side command appends only)."""
        L_, h = lib(), self._h
        rm, af, ao = L_.okb_window_remove_frame, L_.okb_window_add_frame, L_.okb_window_add_observations
        for win, last, pose, sb, t, smp, n, n_obs, obs, _ in prepared:
            rc = rm(h, win, last, last) or af(h, win, pose, sb, t, smp, n) or ao(h, win, n_obs, obs)
            if rc:
                self._check(rc)

    def debug_phase_us(self, win):
        out = np.zeros(16)
        self._check(lib().okb_debug_phase_ns(self._h, int(win), _p(out)))
        names = ["dense_terms", "gather", "assemble", "cholesky", "substitution", "backsub", "dogleg", "_",
                 "p8", "p9", "p10", "p11", "p12", "p13", "p14", "p15"]   # OKB_SCHUR_PROF / OKB_CHOL_PROF builds: cycles
        return {n: v * 1e-3 for n, v in zip(names, out)}

    def debug_schur_plan(self, first=0, count=1):
        out = np.zeros(3, dtype=np.int32)
        self._check(lib().okb_debug_schur_plan(self._h, int(first), int(count), _p(out)))
        return {"acc_smem": bool(out[0]), "threads": int(out[1]), "smem_bytes": int(out[2])}

    def debug_imu_cache(self, win, term):
        ref = np.zeros(9)
        v, r = C.c_int32(0), C.c_int32(0)
        self._check(lib().okb_debug_imu_cache(self._h, int(win), int(term), _p(ref), C.byref(v), C.byref(r)))
        return ref, v.value, r.value

    def debug_imu_terms(self, win, first_term, n_terms):
        """okb_debug_imu_terms: (H30 [n][30][30], g30 [n][30], cost [n]) of the window's last k_imu launch (stale after
        an edit)."""
        out = np.zeros((int(n_terms), abi.IMU_TERM_OUT))
        self._check(lib().okb_debug_imu_terms(self._h, int(win), int(first_term), int(n_terms), _p(out)))
        return out[:, :900].reshape(-1, 30, 30), out[:, 900:930].copy(), out[:, 930].copy()

    def h2d_bytes(self, win):
        f = lib().okb_window_h2d_bytes
        f.restype = C.c_int64
        return int(f(self._h, int(win)))

    def reset(self, first=0, count=1):
        self._check(lib().okb_window_reset(self._h, int(first), int(count)))

    @staticmethod
    def _options(max_iterations, min_iterations, time_limit_s, use_cauchy_loss):
        o = abi.SolveOptions()
        o.max_iterations, o.min_iterations, o.time_limit_s, o.use_cauchy_loss = (max_iterations, min_iterations,
                                                                                time_limit_s, use_cauchy_loss)
        return o

    def optimize(self, first=0, count=1, max_iterations=10, min_iterations=0, time_limit_s=-1.0, use_cauchy_loss=1):
        o = self._options(max_iterations, min_iterations, time_limit_s, use_cauchy_loss)
        out = (abi.Summary * count)()
        self._check(lib().okb_optimize(self._h, int(first), int(count), C.byref(o), out))
        return [s.as_dict() for s in out]

    def optimize_async(self, first=0, count=1, max_iterations=10, min_iterations=0, time_limit_s=-1.0,
                       use_cauchy_loss=1):
        o = self._options(max_iterations, min_iterations, time_limit_s, use_cauchy_loss)
        self._check(lib().okb_optimize_async(self._h, int(first), int(count), C.byref(o)))

    def optimize_finish(self, first=0, count=1):
        out = (abi.Summary * count)()
        self._check(lib().okb_optimize_finish(self._h, int(first), int(count), out))
        return [s.as_dict() for s in out]

    @staticmethod
    def _slot_list(slots):
        arr = (C.c_int32 * len(slots))(*[int(x) for x in slots])
        return len(slots), arr

    def optimize_slots(self, slots, max_iterations=10, min_iterations=0, time_limit_s=-1.0, use_cauchy_loss=1):
        """okb_optimize_slots: one batched solve of the listed slots (any order); summaries in list order."""
        o = self._options(max_iterations, min_iterations, time_limit_s, use_cauchy_loss)
        n, arr = self._slot_list(slots)
        out = (abi.Summary * max(n, 1))()
        self._check(lib().okb_optimize_slots(self._h, n, arr, C.byref(o), out))
        return [s.as_dict() for s in out[:n]]

    def optimize_slots_async(self, slots, max_iterations=10, min_iterations=0, time_limit_s=-1.0, use_cauchy_loss=1):
        o = self._options(max_iterations, min_iterations, time_limit_s, use_cauchy_loss)
        n, arr = self._slot_list(slots)
        self._check(lib().okb_optimize_slots_async(self._h, n, arr, C.byref(o)))

    def optimize_slots_finish(self, slots):
        n, arr = self._slot_list(slots)
        out = (abi.Summary * max(n, 1))()
        self._check(lib().okb_optimize_slots_finish(self._h, n, arr, out))
        return [s.as_dict() for s in out[:n]]

    def download(self, win, with_quality=True, dims=None):
        """dims = (n_poses, n_speed_bias, n_landmarks) when the window was changed incrementally since its upload."""
        if dims is None:
            w = self._windows[win]
            dims = (len(w.poses), len(w.speed_bias), len(w.landmarks))
        poses, sb, lms = np.zeros((dims[0], 7)), np.zeros((dims[1], 9)), np.zeros((dims[2], 4))
        q = np.zeros(dims[2]) if with_quality else None
        self._check(lib().okb_window_download(self._h, int(win), _p(poses), _p(sb), _p(lms), _p(q)))
        return dict(poses=poses, speed_bias=sb, landmarks=lms, quality=q)

    def upload_batch(self, first, windows, host_threads=0, descs=None):
        """okb_window_upload_batch; `descs` (from make_descs) may be cached by the caller while the host arrays live."""
        if descs is None:
            descs = self.make_descs(windows)
        self._check(lib().okb_window_upload_batch(self._h, int(first), len(windows), descs, int(host_threads)))
        for i, w in enumerate(windows):
            self._windows[first + i] = w

    @staticmethod
    def make_descs(windows):
        arr = (abi.WindowDesc * len(windows))()
        for i, w in enumerate(windows):
            arr[i] = w.desc()
        arr._keep = list(windows)
        return arr

    def alloc_outputs(self, first, count):
        """Host buffers for download_batch plus the pointer tables over them."""
        return self.alloc_slot_outputs(range(first, first + count))

    def alloc_slot_outputs(self, slots):
        """Host buffers for download_slots (list order) plus the pointer tables over them."""
        outs = []
        for i in slots:
            w = self._windows[i]
            outs.append(dict(poses=np.zeros_like(w.poses), speed_bias=np.zeros_like(w.speed_bias),
                             landmarks=np.zeros_like(w.landmarks), quality=np.zeros(len(w.landmarks))))
        PP = C.POINTER(C.c_double) * len(outs)
        tables = [PP(*[o[k].ctypes.data_as(C.POINTER(C.c_double)) for o in outs])
                  for k in ("poses", "speed_bias", "landmarks", "quality")]
        return outs, tables

    def download_batch(self, first, count, out=None):
        outs, tables = out if out is not None else self.alloc_outputs(first, count)
        self._check(lib().okb_window_download_batch(self._h, int(first), int(count), *tables))
        return outs

    def download_slots(self, slots, out=None):
        """okb_window_download_slots: the estimates of the listed slots (any order), in list order.  `out` as from
        alloc_slot_outputs(slots) (the buffers follow each slot's uploaded window shape)."""
        outs, tables = out if out is not None else self.alloc_slot_outputs(slots)
        n, arr = self._slot_list(slots)
        self._check(lib().okb_window_download_slots(self._h, n, arr, *tables))
        return outs

    # ---------------------------------------------------------------- single-block hooks
    def eval_reprojection(self, cam, pose, lm, ext, z, sqrt_info):
        pose, lm, ext, z, sqrt_info = map(_f64, (pose, lm, ext, z, sqrt_info))
        n = len(pose)
        cam_arr = np.array([cam], dtype=abi.camera_dtype)
        r, J0, J1, J2 = np.zeros((n, 2)), np.zeros((n, 2, 6)), np.zeros((n, 2, 3)), np.zeros((n, 2, 6))
        self._check(lib().okb_eval_reprojection(self._h, n, _p(cam_arr), _p(pose), _p(lm), _p(ext), _p(z),
                                                _p(sqrt_info), _p(r), _p(J0), _p(J1), _p(J2)))
        return r, J0, J1, J2

    def eval_imu(self, params, samples, t0_ns, t1_ns, pose0, sb0, pose1, sb1, sb_ref=None):
        a = [_f64(x) for x in (pose0, sb0, pose1, sb1)]
        ref = _f64(sb_ref) if sb_ref is not None else None
        samples = np.ascontiguousarray(samples)
        r = np.zeros(15)
        J = [np.zeros((15, 6)), np.zeros((15, 9)), np.zeros((15, 6)), np.zeros((15, 9))]
        sq = np.zeros((15, 15))
        rc = lib().okb_eval_imu(self._h, C.byref(params), _p(samples), len(samples), C.c_int64(int(t0_ns)),
                                C.c_int64(int(t1_ns)), *[_p(x) for x in a], _p(ref), _p(r), *[_p(j) for j in J], _p(sq))
        if rc < 0:
            self._check(rc)
        return r, J, sq, rc

    def imu_propagate(self, params, samples, t0_ns, t1_ns, pose, sb, want_cov=True, want_jac=True):
        pose, sb = np.array(pose, dtype=np.float64), np.array(sb, dtype=np.float64)
        samples = np.ascontiguousarray(samples)
        P, F = np.zeros((15, 15)), np.zeros((15, 15))
        n = C.c_int(0)
        self._check(lib().okb_imu_propagate(self._h, C.byref(params), _p(samples), len(samples), C.c_int64(int(t0_ns)),
                                            C.c_int64(int(t1_ns)), _p(pose), _p(sb), _p(P) if want_cov else None,
                                            _p(F) if want_jac else None, C.byref(n)))
        return n.value, pose, sb, P, F

    def imu_propagate_batch(self, jobs):
        """okb_imu_propagate_batch.  jobs: (params, samples, t0_ns, t1_ns, pose, sb[, want_cov[, want_jac]]) tuples, as
        the arguments of imu_propagate.  Returns per job what imu_propagate returns."""
        arr = (abi.PropagateJob * max(len(jobs), 1))()
        out, keep = [], []
        for j, job in zip(arr, jobs):
            params, samples, t0_ns, t1_ns, pose, sb = job[:6]
            want_cov, want_jac = (tuple(job[6:]) + (True, True))[:2]
            pose, sb = np.array(pose, dtype=np.float64), np.array(sb, dtype=np.float64)
            samples = np.ascontiguousarray(samples)
            P, F, n = np.zeros((15, 15)), np.zeros((15, 15)), np.zeros(1, np.int32)
            j.params, j.samples, j.n_samples = C.pointer(params), samples.ctypes.data, len(samples)
            j.t0_ns, j.t1_ns = int(t0_ns), int(t1_ns)
            j.pose, j.speed_bias = abi.dptr(pose), abi.dptr(sb)
            j.covariance, j.jacobian = abi.dptr(P) if want_cov else None, abi.dptr(F) if want_jac else None
            j.n_used = n.ctypes.data_as(C.POINTER(C.c_int32))
            keep.append(samples)
            out.append((n, pose, sb, P, F))
        self._check(lib().okb_imu_propagate_batch(self._h, len(jobs), arr))
        return [(int(n[0]), pose, sb, P, F) for n, pose, sb, P, F in out]

    def eval_pose_error(self, meas, sqrt_info, pose):
        r, J = np.zeros(6), np.zeros((6, 6))
        self._check(lib().okb_eval_pose_error(self._h, _p(_f64(meas)), _p(_f64(sqrt_info)), _p(_f64(pose)), _p(r), _p(J)))
        return r, J

    def eval_speed_bias_error(self, meas, sqrt_info, sb):
        r, J = np.zeros(9), np.zeros((9, 9))
        self._check(lib().okb_eval_speed_bias_error(self._h, _p(_f64(meas)), _p(_f64(sqrt_info)), _p(_f64(sb)), _p(r),
                                                    _p(J)))
        return r, J

    def eval_relative_pose(self, sqrt_info, pose0, pose1):
        r, J0, J1 = np.zeros(6), np.zeros((6, 6)), np.zeros((6, 6))
        self._check(lib().okb_eval_relative_pose(self._h, _p(_f64(sqrt_info)), _p(_f64(pose0)), _p(_f64(pose1)), _p(r),
                                                 _p(J0), _p(J1)))
        return r, J0, J1

    def eval_marginalization(self, marg, x):
        m = abi.MargPrior()
        m.n, m.n_blocks = int(marg["J"].shape[0]), len(marg["block_kind"])
        m.block_kind = marg["block_kind"].ctypes.data_as(C.POINTER(C.c_int32))
        m.block_idx = marg["block_idx"].ctypes.data_as(C.POINTER(C.c_uint32))
        m.x0, m.J, m.e0 = abi.dptr(marg["x0"]), abi.dptr(marg["J"]), abi.dptr(marg["e0"])
        r, J = np.zeros(m.n), np.zeros((m.n, m.n))
        self._check(lib().okb_eval_marginalization(self._h, C.byref(m), _p(_f64(x)), _p(r), _p(J)))
        return r, J

    # ---------------------------------------------------------------- frontend path
    def hamming_match(self, A, B, skipA=None, skipB=None, threshold=60.0, num_best=4, use_ratio=False,
                      ratio_threshold=3.0):
        A = np.ascontiguousarray(A, dtype=np.uint8)
        B = np.ascontiguousarray(B, dtype=np.uint8)
        nA, nB, nbytes = A.shape[0], B.shape[0], A.shape[1]
        topk = np.zeros((nA, num_best), abi.pair_dtype)
        pairs = np.zeros(nB, abi.pair_dtype)
        sa = np.ascontiguousarray(skipA, dtype=np.uint8) if skipA is not None else None
        sb = np.ascontiguousarray(skipB, dtype=np.uint8) if skipB is not None else None
        self._check(lib().okb_hamming_match(self._h, _p(A), nA, _p(B), nB, nbytes, _p(sa), _p(sb), C.c_float(threshold),
                                            num_best, int(use_ratio), C.c_float(ratio_threshold), _p(topk), _p(pairs)))
        return dict(topk=topk, pairs=pairs)

    def hamming_match_gated(self, A, B, gate, skipA=None, skipB=None, threshold=60.0, num_best=4, use_ratio=False, ratio_threshold=3.0):
        """okb_hamming_match_gated; gate from abi.make_match_gate."""
        A = np.ascontiguousarray(A, dtype=np.uint8)
        B = np.ascontiguousarray(B, dtype=np.uint8)
        nA, nB, nbytes = A.shape[0], B.shape[0], A.shape[1]
        topk = np.zeros((nA, num_best), abi.pair_dtype)
        pairs = np.zeros(nB, abi.pair_dtype)
        sa = np.ascontiguousarray(skipA, dtype=np.uint8) if skipA is not None else None
        sb = np.ascontiguousarray(skipB, dtype=np.uint8) if skipB is not None else None
        self._check(lib().okb_hamming_match_gated(self._h, _p(A), nA, _p(B), nB, nbytes, _p(sa), _p(sb), C.c_float(threshold), num_best,
                                                  int(use_ratio), C.c_float(ratio_threshold), C.byref(gate), _p(topk), _p(pairs)))
        return dict(topk=topk, pairs=pairs)

    def hamming_candidates(self, A, B, threshold=60.0, cap=None):
        A = np.ascontiguousarray(A, dtype=np.uint8)
        B = np.ascontiguousarray(B, dtype=np.uint8)
        nA, nB, nbytes = A.shape[0], B.shape[0], A.shape[1]
        cap = cap or max(nA * nB, 1)
        row_ptr = np.zeros(nA + 1, np.uint32)
        col = np.zeros(cap, np.uint32)
        dist = np.zeros(cap, np.uint16)
        rc = lib().okb_hamming_candidates(self._h, _p(A), nA, _p(B), nB, nbytes, C.c_float(threshold), _p(row_ptr),
                                          _p(col), _p(dist), cap)
        self._check(rc)
        n = int(row_ptr[-1])
        return row_ptr, col[:n].copy(), dist[:n].copy()

    def detect_describe(self, img, cam, R_CW, uniformity_radius=40.0, absolute_threshold=800.0, max_keypoints=400,
                        desc_bytes=48, rotation_invariance=True, cam_slot=0):
        img = np.ascontiguousarray(img, dtype=np.uint8)
        h, w = img.shape
        prm = abi.DetectParams()
        prm.uniformity_radius, prm.absolute_threshold = uniformity_radius, absolute_threshold
        prm.max_keypoints, prm.desc_bytes, prm.rotation_invariance = max_keypoints, desc_bytes, int(rotation_invariance)
        cam_arr = np.array([cam], dtype=abi.camera_dtype)
        R = _f64(np.asarray(R_CW).reshape(9))
        kps = np.zeros(max_keypoints, abi.keypoint_dtype)
        desc = np.zeros((max_keypoints, desc_bytes), np.uint8)
        n = C.c_int(0)
        self._check(lib().okb_detect_describe(self._h, int(cam_slot), _p(img), w, h, img.strides[0], _p(cam_arr), _p(R),
                                              C.byref(prm), _p(kps), _p(desc), max_keypoints, C.byref(n)))
        return kps[:n.value].copy(), desc[:n.value].copy()

    @staticmethod
    def _detect_params(uniformity_radius, absolute_threshold, max_keypoints, desc_bytes, rotation_invariance):
        prm = abi.DetectParams()
        prm.uniformity_radius, prm.absolute_threshold = uniformity_radius, absolute_threshold
        prm.max_keypoints, prm.desc_bytes, prm.rotation_invariance = max_keypoints, desc_bytes, int(rotation_invariance)
        return prm

    @staticmethod
    def _image_descs(imgs, cams, R_CWs):
        """okb_image_desc array over 2-D uint8 images (rows may be strided) and the arrays it points into."""
        descs = (abi.ImageDesc * max(len(imgs), 1))()
        keep = []
        for i, (img, cam, R) in enumerate(zip(imgs, cams, R_CWs)):
            img = np.asarray(img, dtype=np.uint8)
            if img.strides[1] != 1:
                img = np.ascontiguousarray(img)
            keep.append(img)
            d = descs[i]
            d.img = img.ctypes.data
            d.height, d.width = img.shape
            d.stride = img.strides[0]
            ca = np.array([cam], abi.camera_dtype)      # held until the copy: callers may run on several threads
            C.memmove(C.addressof(d.cam), ca.ctypes.data, C.sizeof(abi.Camera))
            for k, v in enumerate(np.asarray(R, dtype=np.float64).reshape(9)):
                d.R_CW[k] = float(v)
        return descs, keep

    def detect_describe_batch(self, imgs, cams, R_CWs, uniformity_radius=40.0, absolute_threshold=800.0, max_keypoints=400,
                              desc_bytes=48, rotation_invariance=True, host_threads=0, return_status=False):
        """okb_detect_describe_batch: one (keypoints, descriptors) per image, each equal to detect_describe on it.
        `imgs` are 2-D uint8 arrays (rows may be strided).  With return_status the call returns (results, status) instead
        of raising OKB_ERR_CAPACITY; an image over the candidate capacity then gives None."""
        n = len(imgs)
        prm = self._detect_params(uniformity_radius, absolute_threshold, max_keypoints, desc_bytes, rotation_invariance)
        descs, keep = self._image_descs(imgs, cams, R_CWs)
        kps = np.zeros((n, max_keypoints), abi.keypoint_dtype)
        desc = np.zeros((n, max_keypoints, desc_bytes), np.uint8)
        n_out = np.zeros(n, np.int32)
        rc = lib().okb_detect_describe_batch(self._h, n, descs, C.byref(prm), _p(kps), _p(desc), max_keypoints, _p(n_out),
                                             int(host_threads))
        if rc != 0 and not (return_status and rc == abi.OKB_ERR_CAPACITY):
            self._check(rc)
        out = [(kps[i, :m].copy(), desc[i, :m].copy()) if m >= 0 else None for i, m in enumerate(n_out.tolist())]
        return (out, rc) if return_status else out

    def detect_describe_store_batch(self, jobs, uniformity_radius=40.0, absolute_threshold=800.0, max_keypoints=400,
                                    desc_bytes=48, rotation_invariance=True, host_threads=0, return_status=False, max_out=None):
        """okb_detect_describe_store_batch.  jobs: dicts with win, feat_slot, imgs, cams, R_CWs (one image per camera, as
        detect_describe_batch takes them) and optionally want_desc (True).  Returns one list per job of (keypoints,
        descriptors or None) per camera, each equal to detect_describe_batch on that image; the images' features are then
        in the store entries (win, feat_slot, camera).  return_status as detect_describe_batch."""
        max_out = max_keypoints if max_out is None else int(max_out)
        prm = self._detect_params(uniformity_radius, absolute_threshold, max_keypoints, desc_bytes, rotation_invariance)
        arr = (abi.DetectStoreJob * max(len(jobs), 1))()
        outs, keep = [], []
        for i, j in enumerate(jobs):
            n = len(j["imgs"])
            descs, k = self._image_descs(j["imgs"], j["cams"], j["R_CWs"])
            o = dict(kp=np.zeros((max(n, 1), max_out), abi.keypoint_dtype), n=np.zeros(max(n, 1), np.int32),
                     desc=np.zeros((max(n, 1), max_out, desc_bytes), np.uint8) if j.get("want_desc", True) else None)
            keep += [descs, k]
            t = arr[i]
            t.win, t.feat_slot, t.n_cams = int(j["win"]), int(j["feat_slot"]), n
            t.images = C.cast(descs, C.POINTER(abi.ImageDesc))
            t.out_kp, t.out_desc = o["kp"].ctypes.data, o["desc"].ctypes.data if o["desc"] is not None else None
            t.n_out = o["n"].ctypes.data_as(C.POINTER(C.c_int32))
            outs.append((o, n))
        rc = lib().okb_detect_describe_store_batch(self._h, len(jobs), arr, C.byref(prm), max_out, int(host_threads))
        if rc != 0 and not (return_status and rc == abi.OKB_ERR_CAPACITY):
            self._check(rc)
        res = [[(o["kp"][c, :m].copy(), o["desc"][c, :m].copy() if o["desc"] is not None else None) if m >= 0 else None
                for c, m in enumerate(o["n"][:n].tolist())] for o, n in outs]
        return (res, rc) if return_status else res

    def debug_features(self, win, feat_slot, cam):
        """okb_debug_features: the committed store entry (win, feat_slot, cam) as a dict of n, kp [n][2], size, desc,
        lm_slot and observed (n = -1: no image; the arrays are then empty)."""
        N, D = self._feat_shape[int(win)]
        n = C.c_int32(0)
        kp, size = np.zeros((N, 2)), np.zeros(N)
        desc, lm, ob = np.zeros((N, D), np.uint8), np.zeros(N, np.int32), np.zeros(N, np.uint8)
        self._check(lib().okb_debug_features(self._h, int(win), int(feat_slot), int(cam), C.byref(n), _p(kp), _p(size), _p(desc),
                                             _p(lm), _p(ob)))
        m = max(n.value, 0)
        return dict(n=n.value, kp=kp[:m].copy(), size=size[:m].copy(), desc=desc[:m].copy(), lm_slot=lm[:m].copy(),
                    observed=ob[:m].copy())

    @staticmethod
    def make_match_job(A, B, skipA=None, skipB=None, threshold=60.0, num_best=4, use_ratio=False, gate=None, want_topk=True):
        """One okb_match_job over numpy arrays; its output arrays are job.topk (or None) and job.pairs."""
        A = np.ascontiguousarray(A, dtype=np.uint8)
        B = np.ascontiguousarray(B, dtype=np.uint8)
        sa = np.ascontiguousarray(skipA, dtype=np.uint8) if skipA is not None else None
        sb = np.ascontiguousarray(skipB, dtype=np.uint8) if skipB is not None else None
        j = abi.MatchJob()
        j.A, j.B = A.ctypes.data, B.ctypes.data
        j.skipA = sa.ctypes.data if sa is not None else None
        j.skipB = sb.ctypes.data if sb is not None else None
        j.nA, j.nB, j.threshold, j.num_best, j.use_ratio = A.shape[0], B.shape[0], threshold, num_best, int(use_ratio)
        if gate is not None:
            j.gate = C.pointer(gate)
        j.topk = np.zeros((A.shape[0], num_best), abi.pair_dtype) if want_topk else None
        j.pairs = np.zeros(B.shape[0], abi.pair_dtype)
        j.out_topk = j.topk.ctypes.data if want_topk else None
        j.out_pairs = j.pairs.ctypes.data
        j._keep = (A, B, sa, sb, gate)
        return j

    # ---- feature store + 3D-2D tracking (okb_window_reserve_features .. okb_track_3d2d_batch)
    def reserve_features(self, win, max_feature_frames, max_cameras, max_keypoints, desc_bytes=48):
        self._check(lib().okb_window_reserve_features(self._h, int(win), int(max_feature_frames), int(max_cameras),
                                                      int(max_keypoints), int(desc_bytes)))
        self._feat = getattr(self, "_feat", {})
        self._feat[int(win)] = int(max_keypoints)
        self._feat_shape = getattr(self, "_feat_shape", {})
        self._feat_shape[int(win)] = (int(max_keypoints), int(desc_bytes))

    def set_features(self, win, feat_slot, cam, kp, desc, lm_slot=None, observed=None):
        """okb_window_set_features: kp is a keypoint_dtype array or an [n][3] array of (x, y, size)."""
        kp = np.asarray(kp)
        if kp.dtype != abi.keypoint_dtype:
            k = np.zeros(len(kp), abi.keypoint_dtype)
            if len(kp):
                k["x"], k["y"], k["size"] = kp[:, 0], kp[:, 1], kp[:, 2]
            kp = k
        kp = np.ascontiguousarray(kp)
        desc = np.ascontiguousarray(desc, dtype=np.uint8)
        lm = np.ascontiguousarray(lm_slot, dtype=np.int32) if lm_slot is not None else None
        ob = np.ascontiguousarray(observed, dtype=np.uint8) if observed is not None else None
        self._check(lib().okb_window_set_features(self._h, int(win), int(feat_slot), int(cam), len(kp), _p(kp), _p(desc), _p(lm), _p(ob)))

    def set_feature_landmarks(self, win, feat_slot, cam, kp_idx, lm_slot, observed):
        k = np.ascontiguousarray(kp_idx, dtype=np.int32)
        lm = np.ascontiguousarray(lm_slot, dtype=np.int32)
        ob = np.ascontiguousarray(observed, dtype=np.uint8)
        self._check(lib().okb_window_set_feature_landmarks(self._h, int(win), int(feat_slot), int(cam), len(k), _p(k), _p(lm), _p(ob)))

    def clear_features(self, win, feat_slot):
        self._check(lib().okb_window_clear_features(self._h, int(win), int(feat_slot)))

    def set_landmark_initialized(self, win, idx, flags):
        i = np.ascontiguousarray(idx, dtype=np.uint32)
        f = np.ascontiguousarray(flags, dtype=np.uint8)
        self._check(lib().okb_window_set_landmark_initialized(self._h, int(win), len(i), _p(i), _p(f)))

    def track_3d2d_batch(self, jobs):
        """okb_track_3d2d_batch.  jobs: dicts with win, pose_b, sb_b (-1: none), feat_slot_b, rounds [(feat_slot_a, cam_a,
        cam_b), ...] and optionally threshold (60) and num_best (4).  Returns one dict per job: assoc (track_assoc_dtype,
        call order), num_matches / num_uncertain per round, uninit (landmark slots cleared, in order)."""
        arr = (abi.TrackJob * max(len(jobs), 1))()
        outs = []
        for i, j in enumerate(jobs):
            rounds = list(j["rounds"])
            cap = max(len(rounds) * getattr(self, "_feat", {}).get(int(j["win"]), 0), 1)
            o = dict(rounds=(abi.TrackRound * max(len(rounds), 1))(), assoc=np.zeros(cap, abi.track_assoc_dtype),
                     n_assoc=C.c_int32(0), num_matches=np.zeros(max(len(rounds), 1), np.int32),
                     num_uncertain=np.zeros(max(len(rounds), 1), np.int32), uninit=np.zeros(cap, np.uint32), n_uninit=C.c_int32(0))
            for r, (fa, ca, cb) in enumerate(rounds):
                o["rounds"][r].feat_slot_a, o["rounds"][r].cam_a, o["rounds"][r].cam_b = int(fa), int(ca), int(cb)
            t = arr[i]
            t.win, t.pose_b, t.sb_b, t.feat_slot_b = int(j["win"]), int(j["pose_b"]), int(j.get("sb_b", -1)), int(j["feat_slot_b"])
            t.threshold, t.num_best, t.n_rounds = float(j.get("threshold", 60.0)), int(j.get("num_best", 4)), len(rounds)
            t.rounds = C.cast(o["rounds"], C.POINTER(abi.TrackRound))
            t.assoc, t.assoc_cap, t.n_assoc = o["assoc"].ctypes.data, cap, C.pointer(o["n_assoc"])
            t.num_matches = o["num_matches"].ctypes.data_as(C.POINTER(C.c_int32))
            t.num_uncertain = o["num_uncertain"].ctypes.data_as(C.POINTER(C.c_int32))
            t.uninit, t.uninit_cap, t.n_uninit = o["uninit"].ctypes.data_as(C.POINTER(C.c_uint32)), cap, C.pointer(o["n_uninit"])
            outs.append((o, len(rounds)))
        self._check(lib().okb_track_3d2d_batch(self._h, len(jobs), arr))
        return [dict(assoc=o["assoc"][:o["n_assoc"].value].copy(), num_matches=o["num_matches"][:n].copy(),
                     num_uncertain=o["num_uncertain"][:n].copy(), uninit=o["uninit"][:o["n_uninit"].value].copy()) for o, n in outs]

    def stereo_init_batch(self, jobs):
        """okb_stereo_init_batch.  jobs: dicts with win, pose, feat_slot, cam_a, cam_b and optionally threshold (60) and
        num_best (4).  Returns one stereo_match_dtype array per job, in the reference's setBestMatch order."""
        arr = (abi.StereoJob * max(len(jobs), 1))()
        outs = []
        for i, j in enumerate(jobs):
            cap = max(getattr(self, "_feat", {}).get(int(j["win"]), 0), 1)
            o = dict(out=np.zeros(cap, abi.stereo_match_dtype), n=C.c_int32(0))
            t = arr[i]
            t.win, t.pose, t.feat_slot, t.cam_a, t.cam_b = (int(j[k]) for k in ("win", "pose", "feat_slot", "cam_a", "cam_b"))
            t.threshold, t.num_best = float(j.get("threshold", 60.0)), int(j.get("num_best", 4))
            t.out, t.out_cap, t.n_out = o["out"].ctypes.data, int(j.get("out_cap", cap)), C.pointer(o["n"])
            outs.append(o)
        self._check(lib().okb_stereo_init_batch(self._h, len(jobs), arr))
        return [o["out"][:o["n"].value].copy() for o in outs]

    def match2d2d_batch(self, jobs):
        """okb_match2d2d_batch.  jobs: dicts with win, pose_a, feat_slot_a, cam_a, pose_b, feat_slot_b, cam_b and
        optionally sb_current (-1), threshold (60) and num_best (4).  Returns one stereo_match_dtype array per job, in
        the reference's setBestMatch order."""
        arr = (abi.Match2D2DJob * max(len(jobs), 1))()
        outs = []
        for i, j in enumerate(jobs):
            cap = max(getattr(self, "_feat", {}).get(int(j["win"]), 0), 1)
            o = dict(out=np.zeros(cap, abi.stereo_match_dtype), n=C.c_int32(0))
            t = arr[i]
            (t.win, t.pose_a, t.feat_slot_a, t.cam_a, t.pose_b, t.feat_slot_b, t.cam_b) = (
                int(j[k]) for k in ("win", "pose_a", "feat_slot_a", "cam_a", "pose_b", "feat_slot_b", "cam_b"))
            t.sb_current = int(j.get("sb_current", -1))
            t.threshold, t.num_best = float(j.get("threshold", 60.0)), int(j.get("num_best", 4))
            t.out, t.out_cap, t.n_out = o["out"].ctypes.data, int(j.get("out_cap", cap)), C.pointer(o["n"])
            outs.append(o)
        self._check(lib().okb_match2d2d_batch(self._h, len(jobs), arr))
        return [o["out"][:o["n"].value].copy() for o in outs]

    def keyframe_overlap_batch(self, jobs):
        """okb_keyframe_overlap_batch.  jobs: dicts with win, feat_slot, n_cams and optionally overlap_threshold (0.6)
        and matching_ratio_threshold (0.2), passed as floats.  Returns one dict per job: need_keyframe (bool), overlap and
        ratio (the maxima) and cams (one dict of okb_keyframe_cam's fields per camera)."""
        arr = (abi.KeyframeJob * max(len(jobs), 1))()
        outs = []
        for i, j in enumerate(jobs):
            n = int(j["n_cams"])
            o = dict(cams=(abi.KeyframeCam * max(n, 1))(), out=abi.KeyframeResult())
            t = arr[i]
            t.win, t.feat_slot, t.n_cams = int(j["win"]), int(j["feat_slot"]), n
            t.overlap_threshold = float(j.get("overlap_threshold", 0.6))
            t.matching_ratio_threshold = float(j.get("matching_ratio_threshold", 0.2))
            t.cams = C.cast(o["cams"], C.POINTER(abi.KeyframeCam)) if j.get("cams", True) is not None else None
            t.out = C.pointer(o["out"]) if j.get("out", True) is not None else None
            outs.append((o, n))
        self._check(lib().okb_keyframe_overlap_batch(self._h, len(jobs), arr))
        return [dict(need_keyframe=bool(o["out"].need_keyframe), overlap=o["out"].overlap, ratio=o["out"].ratio,
                     cams=[{k: getattr(o["cams"][c], k) for k, _ in abi.KeyframeCam._fields_} for c in range(n)])
                for o, n in outs]

    def ransac_3d2d_batch(self, jobs):
        """okb_ransac_3d2d_batch.  jobs: dicts with win, feat_slot, n_cams, seed and optionally max_iterations (50) and
        threshold (9.0).  Returns one dict per job: okb_ransac_result's fields (T_WS as an array of 7), hyp_inliers (the
        inliers of every hypothesis) and outliers (ransac_outlier_dtype, correspondence order)."""
        arr = (abi.RansacJob * max(len(jobs), 1))()
        outs = []
        for i, j in enumerate(jobs):
            n_hyp = int(j.get("max_iterations", 50))
            cap = int(j.get("outlier_cap", max(int(j["n_cams"]), 0) * getattr(self, "_feat", {}).get(int(j["win"]), 0)))
            o = dict(res=abi.RansacResult(), hyp=np.zeros(max(n_hyp, 1), np.int32), outl=np.zeros(max(cap, 1), abi.ransac_outlier_dtype))
            t = arr[i]
            t.win, t.feat_slot, t.n_cams, t.max_iterations = int(j["win"]), int(j["feat_slot"]), int(j["n_cams"]), n_hyp
            t.threshold, t.seed = float(j.get("threshold", 9.0)), int(j["seed"]) & 0xFFFFFFFFFFFFFFFF
            t.hyp_inliers = o["hyp"].ctypes.data_as(C.POINTER(C.c_int32))
            t.outliers, t.outlier_cap = o["outl"].ctypes.data, cap
            t.out = C.pointer(o["res"]) if j.get("out", True) is not None else None
            outs.append((o, n_hyp))
        self._check(lib().okb_ransac_3d2d_batch(self._h, len(jobs), arr))
        res = []
        for o, n_hyp in outs:
            r = {k: getattr(o["res"], k) for k, _ in abi.RansacResult._fields_ if k not in ("_pad", "T_WS")}
            r["T_WS"] = np.array(o["res"].T_WS[:])
            r["hyp_inliers"] = o["hyp"][:n_hyp].copy()
            r["outliers"] = o["outl"][:r["n_outliers"]].copy()
            res.append(r)
        return res

    def ransac_2d2d_batch(self, jobs):
        """okb_ransac_2d2d_batch.  jobs: dicts with win, pose_b, feat_slot_b, pose_a, feat_slot_a, n_cams, seed and
        optionally initialize_pose (False), max_iterations (50) and threshold (9.0).  Returns one dict per job:
        okb_ransac2d_result's fields (T_WS as an array of 7), cams (one dict of okb_ransac2d_cam's fields per camera, the
        models as arrays: R_rot and R_rel 3x3, t_rel), hyp_inliers ([n_cams][2][max_iterations], problem 0: rotation-only,
        1: five-point) and outliers (ransac2d_outlier_dtype, cameras ascending, then correspondence order)."""
        arr = (abi.Ransac2dJob * max(len(jobs), 1))()
        outs = []
        for i, j in enumerate(jobs):
            n_hyp, n_cams = int(j.get("max_iterations", 50)), int(j["n_cams"])
            cap = int(j.get("outlier_cap", max(n_cams, 0) * getattr(self, "_feat", {}).get(int(j["win"]), 0)))
            o = dict(res=abi.Ransac2dResult(), cams=(abi.Ransac2dCam * max(n_cams, 1))(),
                     hyp=np.zeros(max(n_cams * 2 * n_hyp, 1), np.int32), outl=np.zeros(max(cap, 1), abi.ransac2d_outlier_dtype))
            t = arr[i]
            (t.win, t.pose_b, t.feat_slot_b, t.pose_a, t.feat_slot_a) = (
                int(j[k]) for k in ("win", "pose_b", "feat_slot_b", "pose_a", "feat_slot_a"))
            t.n_cams, t.initialize_pose, t.max_iterations = n_cams, int(bool(j.get("initialize_pose", False))), n_hyp
            t.threshold, t.seed = float(j.get("threshold", 9.0)), int(j["seed"]) & 0xFFFFFFFFFFFFFFFF
            t.hyp_inliers = o["hyp"].ctypes.data_as(C.POINTER(C.c_int32))
            t.cams = C.cast(o["cams"], C.POINTER(abi.Ransac2dCam))
            t.outliers, t.outlier_cap = o["outl"].ctypes.data, cap
            t.out = C.pointer(o["res"]) if j.get("out", True) is not None else None
            outs.append((o, n_hyp, n_cams))
        self._check(lib().okb_ransac_2d2d_batch(self._h, len(jobs), arr))
        res = []
        for o, n_hyp, n_cams in outs:
            r = {k: getattr(o["res"], k) for k, _ in abi.Ransac2dResult._fields_ if k != "T_WS"}
            r["T_WS"] = np.array(o["res"].T_WS[:])
            cams = []
            for c in range(n_cams):
                oc = o["cams"][c]
                d = {k: getattr(oc, k) for k, _ in abi.Ransac2dCam._fields_ if k not in ("R_rot", "R_rel", "t_rel")}
                d["R_rot"] = np.array(oc.R_rot[:]).reshape(3, 3)
                d["R_rel"] = np.array(oc.R_rel[:]).reshape(3, 3)
                d["t_rel"] = np.array(oc.t_rel[:])
                cams.append(d)
            r["cams"] = cams
            r["hyp_inliers"] = o["hyp"][:n_cams * 2 * n_hyp].reshape(n_cams, 2, n_hyp).copy()
            r["outliers"] = o["outl"][:r["n_outliers"]].copy()
            res.append(r)
        return res

    def hamming_match_batch(self, jobs, desc_bytes):
        """okb_hamming_match_batch over `jobs`: make_match_job results, or dicts of its keyword arguments.  Returns one
        dict(topk, pairs) per job, like hamming_match / hamming_match_gated."""
        jobs = [j if isinstance(j, abi.MatchJob) else self.make_match_job(**j) for j in jobs]
        arr = (abi.MatchJob * max(len(jobs), 1))()
        for i, j in enumerate(jobs):
            arr[i] = j
        self._check(lib().okb_hamming_match_batch(self._h, len(jobs), arr, int(desc_bytes)))
        return [dict(topk=j.topk, pairs=j.pairs) for j in jobs]


def matches_from_pairs(pairs, topk, threshold, use_ratio=False, ratio_threshold=3.0):
    """The serial epilogue of DenseMatcher::matchBody (DenseMatcher.hpp(impl):97-122): turns the per-B
    winners into the ordered (A, B, distance) callback list.  Pure bookkeeping on the host side of the
    boundary, exactly where the reference runs setBestMatch."""
    out = []
    for b in range(len(pairs)):
        a, dist = int(pairs[b]["index_a"]), float(pairs[b]["distance"])
        if not dist < threshold:
            continue
        if use_ratio:
            bl = topk[a]
            if bl[1]["index_a"] != -1:
                d0, d1 = float(bl[0]["distance"]), float(bl[1]["distance"])
                if not (d0 == 0 or d1 / d0 > ratio_threshold):
                    continue
        out.append((a, b, dist))
    return out
