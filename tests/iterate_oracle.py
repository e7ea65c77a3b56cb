"""TEST INFRASTRUCTURE ONLY.  ctypes binding of tests/iterate_oracle.cpp: the iterated EKF update (include/sl2b200.h,
sl2_set_stream_iterated) in place of the first update of the CPU oracle's step, on top of the sub-pixel, consensus and
rescue oracles, which it uses unchanged.  The library is compiled on first use, with the oracle's flags, into a
directory under the system's temporary directory named after the hash of its sources, so the repository tree is never
written."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

import subpixel_oracle as so
from oracle import pyoracle as po

_HERE = os.path.dirname(os.path.abspath(__file__))
_ORACLE = os.path.join(os.path.dirname(_HERE), "oracle")
_SRC = os.path.join(_HERE, "iterate_oracle.cpp")
_DEPS = [_SRC] + [os.path.join(_HERE, f) for f in ("subpixel_oracle.cpp", "rescue_oracle.cpp", "consensus_oracle.cpp")]
_lib = None


def _build():
    h = hashlib.sha256()
    for p in _DEPS + sorted(os.path.join(_ORACLE, f) for f in os.listdir(_ORACLE) if f.endswith((".hpp", ".h"))):
        h.update(open(p, "rb").read())
    d = os.path.join(tempfile.gettempdir(), "sl2_iterate_oracle_%d_%s" % (os.getuid(), h.hexdigest()[:16]))
    so_path = os.path.join(d, "libiterate_oracle.so")
    if not os.path.exists(so_path):
        os.makedirs(d, exist_ok=True)
        tmp = so_path + ".%d.tmp" % os.getpid()
        subprocess.check_call([os.environ.get("CXX", "g++"), "-std=c++17", "-O3", "-DNDEBUG", "-ffp-contract=off",
                               "-fPIC", "-shared", "-pthread", "-I", _ORACLE, "-I", _HERE, "-o", tmp, _SRC,
                               "-Wl,-Bsymbolic", "-Wl,--exclude-libs,ALL"])
        os.replace(tmp, so_path)
    return so_path


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(_build())
        for name in ("iter_slam_create", "iter_slam_base", "iter_slam_sub"):
            getattr(L, name).restype = C.c_void_p
        L.iter_slam_base.argtypes = L.iter_slam_sub.argtypes = [C.c_void_p]
        for name in ("iter_slam_destroy", "iter_slam_set", "iter_slam_step", "iter_slam_results", "sub_slam_refined"):
            getattr(L, name).restype = None
        L.iter_slam_set.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_int32, C.c_double]
        L.cons_slam_num_features.restype = C.c_int32
        L.cons_slam_state_size.restype = C.c_int32
        for name in ("cons_slam_add_feature", "cons_slam_set_state", "cons_slam_get_state", "cons_slam_get_features"):
            getattr(L, name).restype = None
        _lib = L
    return _lib


class Slam(so.Slam):
    """The oracle's whole step with the refinement (always on), the consensus (tau), the rescue (chi2) and the iterated
    update 1 (max_iterations, tol).  results() -> (iterations, status, last delta) of the last step."""

    def __init__(self, cfg):
        L = lib()
        self._i = C.c_void_p(L.iter_slam_create(C.byref(cfg)))
        self._r = C.c_void_p(L.iter_slam_sub(self._i))
        self.h = C.c_void_p(L.iter_slam_base(self._i))

    def __del__(self):
        if getattr(self, "_i", None):
            lib().iter_slam_destroy(self._i)
            self._i = self._r = self.h = None

    def set_iterated(self, tau, chi2, max_iterations, tol):
        lib().iter_slam_set(self._i, float(tau), float(chi2), int(max_iterations), float(tol))

    # the base class's calls go to this library (the same cons_slam / sub_slam entry points, compiled in)
    def add_feature(self, y, xp_org, patch):
        y, a = po._f64(y)
        xp_org, b = po._f64(xp_org)
        patch, c = po._u8(patch)
        lib().cons_slam_add_feature(self.h, a, b, c)

    @property
    def num_features(self):
        return lib().cons_slam_num_features(self.h)

    @property
    def n(self):
        return lib().cons_slam_state_size(self.h)

    def set_state(self, x, P):
        x, a = po._f64(x)
        P, b = po._colmajor(P)
        lib().cons_slam_set_state(self.h, a, b)

    def get_state(self):
        x = np.zeros(self.n)
        P = np.zeros((self.n, self.n), order="F")
        lib().cons_slam_get_state(self.h, po._p(x, po.f64p), po._p(P, po.f64p))
        return x, P

    def step(self, frame):
        frame, fp = po._u8(frame)
        lib().iter_slam_step(self._i, fp)

    def features(self):
        nf = self.num_features
        out = dict(label=np.zeros(nf, np.int32), h=np.zeros((nf, 2)), z=np.zeros((nf, 2)),
                   S=np.zeros((nf, 4)), flags=np.zeros(nf, np.uint8),
                   attempted=np.zeros(nf, np.int32), successful=np.zeros(nf, np.int32),
                   select_rank=np.zeros(nf, np.int32))
        lib().cons_slam_get_features(self.h, po._p(out["label"], po.i32p), po._p(out["h"], po.f64p),
                                     po._p(out["z"], po.f64p), po._p(out["S"], po.f64p), po._p(out["flags"], po.u8p),
                                     po._p(out["attempted"], po.i32p), po._p(out["successful"], po.i32p),
                                     po._p(out["select_rank"], po.i32p))
        ref = np.zeros(nf, np.uint8)
        lib().sub_slam_refined(self._r, po._p(ref, po.u8p))
        out["flags"] |= ref << 3
        return out

    def results(self):
        it, st, dl = C.c_int32(), C.c_int32(), C.c_double()
        lib().iter_slam_results(self._i, C.byref(it), C.byref(st), C.byref(dl))
        return it.value, st.value, dl.value


def slam_from_scene(sc, tau, chi2, max_iterations, tol):
    """Slam of a synth.Scene with the consensus at tau, the rescue at chi2 and the iteration at (max_iterations, tol)."""
    cfg = po.make_config(width=sc.width, height=sc.height, fku=sc.cam8[2], fkv=sc.cam8[3], u0=sc.cam8[4],
                         v0=sc.cam8[5], kd1=sc.cam8[6], sd=sc.cam8[7], delta_t=sc.delta_t, n_select=sc.n_select,
                         boxsize=sc.boxsize, search_override=sc.search_override)
    s = Slam(cfg)
    for i in range(sc.n_features):
        s.add_feature(sc.x0[13 + 3 * i:16 + 3 * i], sc.xp_org[i], sc.patches[i])
    s.set_state(sc.x0, sc.P0)
    s.set_iterated(tau, chi2, max_iterations, tol)
    return s
