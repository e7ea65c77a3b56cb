"""ctypes binding of libsl2b200.so — the C ABI declared in include/sl2b200.h.

This module is the Python mirror of the reference-facing boundary: the names and argument
meaning follow MonoSLAM / Kalman (see the header for file:line of each replaced interface).
There is NO fallback: if the CUDA library is missing or no sm_90 device is usable, calls raise.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsl2b200.so")

u8p = C.POINTER(C.c_uint8)
i32p = C.POINTER(C.c_int32)
f64p = C.POINTER(C.c_double)
f32p = C.POINTER(C.c_float)

SL2_MAX_FEATURES = 128
# keys of Context.set_tuning (SL2_TUNE_* of include/sl2b200.h)
TUNE_PDL, TUNE_HP_PIPELINED = 0, 1


class Sl2Config(C.Structure):
    _fields_ = [
        ("device", C.c_int32), ("num_streams", C.c_int32), ("frame_slots", C.c_int32),
        ("width", C.c_int32), ("height", C.c_int32), ("boxsize", C.c_int32),
        ("max_features", C.c_int32), ("number_of_features_to_select", C.c_int32),
        ("search_tile_radius", C.c_int32),
        ("fku", C.c_double), ("fkv", C.c_double), ("u0", C.c_double), ("v0", C.c_double),
        ("kd1", C.c_double), ("sd", C.c_double), ("delta_t", C.c_double),
        ("search_override", C.c_double * 3),
        ("minimum_attempted_measurements_of_feature", C.c_int32),
        ("successful_match_fraction", C.c_double),
        ("cuda_stream", C.c_void_p),
    ]


# every symbol include/sl2b200.h declares (checked by tests/test_abi.py)
EXPORTS = [
    "sl2_default_config", "sl2_create", "sl2_destroy", "sl2_last_error", "sl2_sync", "sl2_version",
    "sl2_set_frame", "sl2_set_frames", "sl2_set_frames_dev", "sl2_set_features",
    "sl2_num_features", "sl2_state_size", "sl2_set_state", "sl2_get_state", "sl2_delete_feature", "sl2_append_feature",
    "sl2_patch_search", "sl2_score_map", "sl2_smoe_search", "sl2_find_best_patch", "sl2_ekf_predict",
    "sl2_predict_measurements", "sl2_make_measurements", "sl2_ekf_update",
    "sl2_ekf_update_measured", "sl2_normalise_state", "sl2_step", "sl2_step_host",
    "sl2_step_host_async", "sl2_wait_slot", "sl2_set_step_groups", "sl2_join", "sl2_set_tuning", "sl2_measure_particles", "sl2_measure_particles_patch",
    "sl2_smoe_search_patch", "sl2_measure_partial_features",
    "sl2_get_features", "sl2_get_feature_jacobians", "sl2_enable_timing", "sl2_last_step_times", "sl2_last_update_times", "sl2_launch_count",
]

_lib = None


class Sl2Error(RuntimeError):
    pass


def load():
    """dlopen libsl2b200.so; raises if it has not been built (no silent fallback)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise Sl2Error("%s not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(there is no CPU fallback)" % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        L.sl2_last_error.restype = C.c_char_p
        L.sl2_last_error.argtypes = [C.c_void_p]
        L.sl2_version.restype = C.c_char_p
        L.sl2_launch_count.restype = C.c_int64
        L.sl2_launch_count.argtypes = [C.c_void_p]
        L.sl2_destroy.restype = None
        L.sl2_destroy.argtypes = [C.c_void_p]
        L.sl2_default_config.restype = None
        L.sl2_set_frame.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_size_t]
        L.sl2_set_frames.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]
        L.sl2_set_frames_dev.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]
        L.sl2_step.argtypes = [C.c_void_p, C.c_int32]
        L.sl2_step_host.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
        L.sl2_step_host_async.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
        L.sl2_wait_slot.argtypes = [C.c_void_p, C.c_int32]
        L.sl2_set_step_groups.argtypes = [C.c_void_p, C.c_int32]
        L.sl2_join.argtypes = [C.c_void_p]
        L.sl2_set_tuning.argtypes = [C.c_void_p, C.c_int32, C.c_int32]
        L.sl2_measure_particles.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, f64p, f64p,
                                            f64p, f64p, C.c_double, f64p, i32p, u8p, u8p, f64p, f64p]
        L.sl2_measure_particles_patch.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, f64p,
                                                  f64p, f64p, f64p, C.c_double, f64p, i32p, u8p, u8p, f64p, f64p]
        L.sl2_smoe_search_patch.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, f64p, f64p,
                                            i32p, i32p, u8p]
        L.sl2_sync.argtypes = [C.c_void_p]
        L.sl2_score_map.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, f64p, f64p, i32p,
                                    f64p, f64p, u8p, C.c_size_t]
        _lib = L
    return _lib


def default_config():
    cfg = Sl2Config()
    load().sl2_default_config(C.byref(cfg))
    return cfg


def _p(a, t):
    return a.ctypes.data_as(t)


def _f64(a):
    a = np.ascontiguousarray(a, dtype=np.float64)
    return a, _p(a, f64p)


def _colmajor(a):
    a = np.asfortranarray(np.asarray(a, np.float64))
    return a, _p(a, f64p)


class Context:
    """One GPU context holding `num_streams` independent camera streams."""

    def __init__(self, cfg):
        self.L = load()
        self.cfg = cfg
        h = C.c_void_p()
        rc = self.L.sl2_create(C.byref(cfg), C.byref(h))
        if rc != 0:
            raise Sl2Error("sl2_create failed (%d): %s" % (rc, self.L.sl2_last_error(None).decode()))
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.L.sl2_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def _ck(self, rc):
        if rc < 0:
            raise Sl2Error("libsl2b200 error %d: %s" % (rc, self.L.sl2_last_error(self.h).decode()))
        return rc

    # ---- frames -------------------------------------------------------------------------------
    def set_frame(self, stream_id, slot, gray):
        gray = np.ascontiguousarray(gray, np.uint8)
        self._ck(self.L.sl2_set_frame(self.h, stream_id, slot, gray.ctypes.data, gray.strides[0]))
        self._ck(self.L.sl2_sync(self.h))

    def set_frames(self, slot, gray):
        """gray: (num_streams, H, W) u8 host array."""
        gray = np.ascontiguousarray(gray, np.uint8)
        assert gray.shape == (self.cfg.num_streams, self.cfg.height, self.cfg.width)
        self._ck(self.L.sl2_set_frames(self.h, slot, gray.ctypes.data))
        self._ck(self.L.sl2_sync(self.h))

    def set_frames_ptr(self, slot, host_ptr):
        self._ck(self.L.sl2_set_frames(self.h, slot, host_ptr))

    def set_frames_dev(self, slot, dev_ptr):
        self._ck(self.L.sl2_set_frames_dev(self.h, slot, dev_ptr))

    # ---- map / state --------------------------------------------------------------------------
    def set_features(self, stream_id, y, xp_org, patches):
        y, yp = _f64(y)
        xp_org, xp = _f64(xp_org)
        patches = np.ascontiguousarray(patches, np.uint8)
        n = patches.shape[0]
        self._ck(self.L.sl2_set_features(self.h, stream_id, n, yp, xp, _p(patches, u8p)))

    def num_features(self, stream_id):
        return self._ck(self.L.sl2_num_features(self.h, stream_id))

    def state_size(self, stream_id):
        return self._ck(self.L.sl2_state_size(self.h, stream_id))

    def set_state(self, stream_id, x, P):
        x, xp = _f64(x)
        P, pp = _colmajor(P)
        self._ck(self.L.sl2_set_state(self.h, stream_id, xp, pp))

    def get_state(self, stream_id):
        n = self.state_size(stream_id)
        x = np.zeros(n)
        P = np.zeros((n, n), order="F")
        self._ck(self.L.sl2_get_state(self.h, stream_id, _p(x, f64p), _p(P, f64p)))
        return x, P

    def append_feature(self, stream_id, y, xp_org, patch, Pcol=None):
        """MonoSLAM::AddNewKnownFeature on the device; Pcol (n+3, 3) column block or None (zeros). Returns the index."""
        y, yp = _f64(y)
        xp, xpp = _f64(xp_org)
        patch = np.ascontiguousarray(patch, np.uint8)
        pc = None
        if Pcol is not None:
            Pcol = np.asfortranarray(Pcol, dtype=np.float64)   # column-major (n + 3) x 3
            pc = Pcol.ctypes.data_as(f64p)
        return self._ck(self.L.sl2_append_feature(self.h, stream_id, yp, xpp, _p(patch, u8p), pc))

    def delete_feature(self, stream_id, index):
        self._ck(self.L.sl2_delete_feature(self.h, stream_id, index))

    # ---- patch search -------------------------------------------------------------------------
    def patch_search(self, stream_id, slot, feat_index, centres, puinv3):
        feat_index = np.ascontiguousarray(feat_index, np.int32)
        centres, cp = _f64(centres)
        puinv3, qp = _f64(puinv3)
        n = feat_index.size
        u = np.zeros(n, np.int32)
        v = np.zeros(n, np.int32)
        found = np.zeros(n, np.uint8)
        best = np.zeros(n, np.float64)
        self._ck(self.L.sl2_patch_search(self.h, stream_id, slot, n, _p(feat_index, i32p), cp, qp,
                                         _p(u, i32p), _p(v, i32p), _p(found, u8p), _p(best, f64p)))
        return u, v, found, best

    def score_map(self, stream_id, slot, feat_index, centre, puinv3, cap=1 << 16):
        centre, cp = _f64(centre)
        puinv3, qp = _f64(puinv3)
        box = np.zeros(6, np.int32)
        corr = np.zeros(cap)
        sd = np.zeros(cap)
        inside = np.zeros(cap, np.uint8)
        self._ck(self.L.sl2_score_map(self.h, stream_id, slot, feat_index, cp, qp, _p(box, i32p),
                                      _p(corr, f64p), _p(sd, f64p), _p(inside, u8p), cap))
        nu, nv = max(0, box[1] - box[0] + 1), max(0, box[3] - box[2] + 1)
        k = nu * nv
        return box, corr[:k].reshape(nu, nv), sd[:k].reshape(nu, nv), inside[:k].reshape(nu, nv)

    def smoe_search(self, stream_id, slot, feat_index, puinv3, centres):
        puinv3, qp = _f64(puinv3)
        centres, cp = _f64(centres)
        K = puinv3.shape[0]
        ru = np.zeros(K, np.int32)
        rv = np.zeros(K, np.int32)
        rf = np.zeros(K, np.uint8)
        self._ck(self.L.sl2_smoe_search(self.h, stream_id, slot, feat_index, K, qp, cp,
                                        _p(ru, i32p), _p(rv, i32p), _p(rf, u8p)))
        return ru, rv, rf

    def smoe_search_patch(self, stream_id, slot, patch, puinv3, centres):
        """SMOE search with a raw template (not a map feature)."""
        patch = np.ascontiguousarray(patch, np.uint8)
        assert patch.shape == (self.cfg.boxsize, self.cfg.boxsize)
        puinv3, qp = _f64(puinv3)
        centres, cp = _f64(centres)
        K = puinv3.shape[0]
        ru, rv, rf = np.zeros(K, np.int32), np.zeros(K, np.int32), np.zeros(K, np.uint8)
        self._ck(self.L.sl2_smoe_search_patch(self.h, stream_id, slot, patch.ctypes.data, K, qp, cp, _p(ru, i32p),
                                              _p(rv, i32p), _p(rf, u8p)))
        return ru, rv, rf

    def measure_particles(self, stream_id, slot, feat_index, h, Sinv3, detS, lam, prune_threshold, prob,
                          patch=None):
        """N2: SMOE search + particle re-weighting of one partially-initialised feature ->
        survivors, prob, z_uv (K,2), found, keep, cumulative, (mean, variance).  With `patch` (B x B u8) the
        template is given directly instead of naming map feature `feat_index`."""
        h, hp = _f64(h)
        Sinv3, sp = _f64(Sinv3)
        detS, dp = _f64(detS)
        lam, lp = _f64(lam)
        prob = np.array(prob, np.float64)
        K = prob.shape[0]
        z = np.zeros((K, 2), np.int32)
        found = np.zeros(K, np.uint8)
        keep = np.zeros(K, np.uint8)
        cum = np.zeros(K)
        mv = np.zeros(2)
        args = (K, hp, sp, dp, lp, float(prune_threshold), _p(prob, f64p), _p(z, i32p), _p(found, u8p),
                _p(keep, u8p), _p(cum, f64p), _p(mv, f64p))
        if patch is None:
            left = self._ck(self.L.sl2_measure_particles(self.h, stream_id, slot, feat_index, *args))
        else:
            patch = np.ascontiguousarray(patch, np.uint8)
            assert patch.shape == (self.cfg.boxsize, self.cfg.boxsize)
            left = self._ck(self.L.sl2_measure_particles_patch(self.h, stream_id, slot, patch.ctypes.data, *args))
        return left, prob, z, found, keep, cum, mv

    def measure_partial_features(self, stream_id, slot, patches, ypi, Pxy, Pyy, lam, prune_threshold, prob, K=None):
        """N2 for F partially-initialised features in one call: device prediction of every particle's ellipse
        (monoslam.cpp:1347-1400), SMOE search with one score map per feature, particle re-weighting.
        patches (F,B,B) u8; ypi (F,6); Pxy (F,13,6); Pyy (F,6,6); lam, prob (F,Kmax); K (F,) particle counts
        (default Kmax).  Returns a dict of arrays."""
        patches = np.ascontiguousarray(patches, np.uint8)
        F = patches.shape[0]
        ypi = np.ascontiguousarray(ypi, np.float64).reshape(F, 6)
        Pxy = np.ascontiguousarray(np.asarray(Pxy, np.float64).reshape(F, 13, 6).transpose(0, 2, 1))  # column-major
        Pyy = np.ascontiguousarray(np.asarray(Pyy, np.float64).reshape(F, 6, 6).transpose(0, 2, 1))
        lam = np.ascontiguousarray(lam, np.float64).reshape(F, -1)
        Kmax = lam.shape[1]
        prob = np.array(prob, np.float64).reshape(F, Kmax)
        K = np.full(F, Kmax, np.int32) if K is None else np.ascontiguousarray(K, np.int32)
        out = {"h": np.zeros((F, Kmax, 2)), "Sinv3": np.zeros((F, Kmax, 3)), "detS": np.zeros((F, Kmax)),
               "z": np.zeros((F, Kmax, 2), np.int32), "found": np.zeros((F, Kmax), np.uint8),
               "keep": np.zeros((F, Kmax), np.uint8), "cumulative": np.zeros((F, Kmax)),
               "mean_var": np.zeros((F, 2)), "left": np.zeros(F, np.int32)}
        self._ck(self.L.sl2_measure_partial_features(
            self.h, stream_id, slot, F, Kmax, _p(K, i32p), C.c_void_p(patches.ctypes.data), _p(ypi, f64p), _p(Pxy, f64p),
            _p(Pyy, f64p), _p(lam, f64p), C.c_double(float(prune_threshold)), _p(prob, f64p), _p(out["h"], f64p),
            _p(out["Sinv3"], f64p), _p(out["detS"], f64p), _p(out["z"], i32p), _p(out["found"], u8p),
            _p(out["keep"], u8p), _p(out["cumulative"], f64p), _p(out["mean_var"], f64p), _p(out["left"], i32p)))
        out["prob"] = prob
        return out

    def find_best_patch(self, stream_id, slot, regions, ubest=-1, vbest=-1):
        """regions (n,4) = (ustart, vstart, ufinish, vfinish) -> u, v (kept at ubest/vbest where the
        reference would not write them), ev."""
        regions = np.ascontiguousarray(regions, np.int32).reshape(-1, 4)
        n = regions.shape[0]
        u = np.full(n, ubest, np.int32)
        v = np.full(n, vbest, np.int32)
        ev = np.zeros(n, np.float64)
        self._ck(self.L.sl2_find_best_patch(self.h, stream_id, slot, n, _p(regions, i32p), _p(u, i32p),
                                            _p(v, i32p), _p(ev, f64p)))
        return u, v, ev

    # ---- EKF ----------------------------------------------------------------------------------
    def ekf_predict(self, stream_id, u3=None):
        if u3 is None:
            self._ck(self.L.sl2_ekf_predict(self.h, stream_id, None))
        else:
            u3, up = _f64(u3)
            self._ck(self.L.sl2_ekf_predict(self.h, stream_id, up))

    def predict_measurements(self, stream_id):
        return self._ck(self.L.sl2_predict_measurements(self.h, stream_id))

    def make_measurements(self, stream_id, slot):
        return self._ck(self.L.sl2_make_measurements(self.h, stream_id, slot))

    def ekf_update(self, stream_id, feat_index, H_xv, H_y, R, nu):
        """H_xv (m,13), H_y (m,3) row-major; R (m/2, 2, 2); nu (m,)."""
        feat_index = np.ascontiguousarray(feat_index, np.int32)
        H_xv, a = _f64(H_xv)
        H_y, b = _f64(H_y)
        R, r = _f64(R)
        nu, nn = _f64(nu)
        self._ck(self.L.sl2_ekf_update(self.h, stream_id, nu.size, _p(feat_index, i32p), a, b, r, nn))

    def ekf_update_measured(self, stream_id):
        self._ck(self.L.sl2_ekf_update_measured(self.h, stream_id))

    def normalise_state(self, stream_id):
        self._ck(self.L.sl2_normalise_state(self.h, stream_id))

    # ---- fused step ---------------------------------------------------------------------------
    def step(self, slot=0):
        self._ck(self.L.sl2_step(self.h, slot))

    def step_host(self, slot, gray_ptr, xv_out_ptr):
        self._ck(self.L.sl2_step_host(self.h, slot, gray_ptr, xv_out_ptr))

    def step_host_async(self, slot, gray_ptr, xv_out_ptr):
        self._ck(self.L.sl2_step_host_async(self.h, slot, gray_ptr, xv_out_ptr))

    def wait_slot(self, slot):
        self._ck(self.L.sl2_wait_slot(self.h, slot))

    def set_step_groups(self, groups):
        self._ck(self.L.sl2_set_step_groups(self.h, groups))

    def join(self):
        self._ck(self.L.sl2_join(self.h))

    def set_tuning(self, key, value):
        """scheduling knob of the fused step (TUNE_* below = SL2_TUNE_* of include/sl2b200.h)"""
        self._ck(self.L.sl2_set_tuning(self.h, int(key), int(value)))

    def sync(self):
        self._ck(self.L.sl2_sync(self.h))

    def enable_timing(self, on=True):
        self._ck(self.L.sl2_enable_timing(self.h, 1 if on else 0))

    def last_step_times(self):
        ms = np.zeros(4, np.float32)
        self._ck(self.L.sl2_last_step_times(self.h, _p(ms, f32p)))
        return ms

    def last_update_times(self):
        """ms of the five EKF update kernels of the last step: hp, chol, solve, syrk, finish"""
        ms = np.zeros(5, np.float32)
        self._ck(self.L.sl2_last_update_times(self.h, _p(ms, f32p)))
        return ms

    def launch_count(self):
        return int(self.L.sl2_launch_count(self.h))

    def feature_jacobians(self, stream_id):
        """Feature::dh_by_dxv_ (nf,26), dh_by_dy_ (nf,6), R_ (nf,4), nu_ (nf,2), column-major like the Eigen members"""
        N = self.cfg.max_features
        J, Jy, R, nu = np.zeros((N, 26)), np.zeros((N, 6)), np.zeros((N, 4)), np.zeros((N, 2))
        nf = self._ck(self.L.sl2_get_feature_jacobians(self.h, stream_id, _p(J, f64p), _p(Jy, f64p), _p(R, f64p),
                                                       _p(nu, f64p)))
        return J[:nf], Jy[:nf], R[:nf], nu[:nf]

    def features(self, stream_id):
        N = self.cfg.max_features
        out = dict(h=np.zeros((N, 2)), z=np.zeros((N, 2)), S=np.zeros((N, 4)),
                   flags=np.zeros(N, np.uint8), attempted=np.zeros(N, np.int32),
                   successful=np.zeros(N, np.int32), select_rank=np.zeros(N, np.int32))
        nf = self._ck(self.L.sl2_get_features(
            self.h, stream_id, _p(out["h"], f64p), _p(out["z"], f64p), _p(out["S"], f64p),
            _p(out["flags"], u8p), _p(out["attempted"], i32p), _p(out["successful"], i32p),
            _p(out["select_rank"], i32p)))
        return {k: v[:nf] for k, v in out.items()}


def config_for_scene(sc, num_streams=1, frame_slots=1, device=0, max_features=None,
                     cuda_stream=None, search_tile_radius=None):
    """sl2_config matching a synth.Scene."""
    cfg = default_config()
    cfg.device = device
    cfg.num_streams = num_streams
    cfg.frame_slots = frame_slots
    cfg.width, cfg.height = sc.width, sc.height
    cfg.boxsize = sc.boxsize
    cfg.max_features = max_features or sc.n_features
    cfg.number_of_features_to_select = sc.n_select
    if search_tile_radius is None:
        rad = sc.meta.get("config", {}).get("radius") or 20
        search_tile_radius = rad
    cfg.search_tile_radius = search_tile_radius
    cfg.fku, cfg.fkv, cfg.u0, cfg.v0, cfg.kd1, cfg.sd = [float(v) for v in sc.cam8[2:8]]
    cfg.delta_t = sc.delta_t
    for i in range(3):
        cfg.search_override[i] = sc.search_override[i]
    if cuda_stream is not None:
        cfg.cuda_stream = cuda_stream
    return cfg


def load_scene(ctx, stream_id, sc):
    """Install a synth.Scene (map + prior) into one stream of a context."""
    n = sc.n_features
    ctx.set_features(stream_id, sc.x0[13:].reshape(n, 3), sc.xp_org, sc.patches)
    ctx.set_state(stream_id, sc.x0, sc.P0)
