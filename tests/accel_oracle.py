"""TEST INFRASTRUCTURE ONLY.  ctypes binding of tests/accel_oracle.cpp: the accelerometer's prediction
(include/sl2b200.h, sl2_set_stream_accel) in place of the CPU oracle's predict when a sample is pending (oracle/ and the
consensus oracle, used unchanged, the consensus off).  The library is compiled on first use, with the oracle's flags, into a
directory under the system's temporary directory named after the hash of its sources, so the repository tree is never
written."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import pyoracle as po

_HERE = os.path.dirname(os.path.abspath(__file__))
_ORACLE = os.path.join(os.path.dirname(_HERE), "oracle")
_SRC = os.path.join(_HERE, "accel_oracle.cpp")
_DEPS = [_SRC, os.path.join(_HERE, "consensus_oracle.cpp")]

u8p, i32p, f64p = po.u8p, po.i32p, po.f64p
_lib = None


def _build():
    h = hashlib.sha256()
    for p in _DEPS + sorted(os.path.join(_ORACLE, f) for f in os.listdir(_ORACLE) if f.endswith((".hpp", ".h"))):
        h.update(open(p, "rb").read())
    d = os.path.join(tempfile.gettempdir(), "sl2_accel_oracle_%d_%s" % (os.getuid(), h.hexdigest()[:16]))
    so = os.path.join(d, "libaccel_oracle.so")
    if not os.path.exists(so):
        os.makedirs(d, exist_ok=True)
        tmp = so + ".%d.tmp" % os.getpid()
        subprocess.check_call([os.environ.get("CXX", "g++"), "-std=c++17", "-O3", "-DNDEBUG", "-ffp-contract=off",
                               "-fPIC", "-shared", "-pthread", "-I", _ORACLE, "-I", _HERE, "-o", tmp, _SRC,
                               "-Wl,-Bsymbolic", "-Wl,--exclude-libs,ALL"])
        os.replace(tmp, so)
    return so


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(_build())
        L.accel_slam_create.restype = C.c_void_p
        L.accel_slam_base.restype = C.c_void_p
        L.accel_slam_base.argtypes = [C.c_void_p]
        L.accel_slam_result.restype = C.c_int32
        for name in ("accel_slam_destroy", "accel_slam_set", "accel_slam_sample", "accel_slam_step"):
            getattr(L, name).restype = None
        L.cons_slam_num_features.restype = C.c_int32
        L.cons_slam_state_size.restype = C.c_int32
        for name in ("cons_slam_add_feature", "cons_slam_set_state", "cons_slam_get_state", "cons_slam_get_features"):
            getattr(L, name).restype = None
        _lib = L
    return _lib


class Slam:
    """The oracle's whole step with the accelerometer's predict: the surface check_streams_against_oracle uses, plus
    set_accel(R_ac, bias, cov, gravity, sd_a), sample(f) (consumed by the next step) and result() -> (a, status)."""

    def __init__(self, cfg):
        self._g = C.c_void_p(lib().accel_slam_create(C.byref(cfg)))
        self.h = C.c_void_p(lib().accel_slam_base(self._g))

    def __del__(self):
        if getattr(self, "_g", None):
            lib().accel_slam_destroy(self._g)
            self._g = self.h = None

    def set_accel(self, R_ac, bias, cov, gravity, sd_a):
        R, a = po._f64(np.asarray(R_ac, np.float64).ravel())
        b, bp = po._f64(np.asarray(bias, np.float64).ravel())
        c, cp = po._f64(np.asarray(cov, np.float64).ravel())
        g, gp = po._f64(np.asarray(gravity, np.float64).ravel())
        lib().accel_slam_set(self._g, a, bp, cp, gp, C.c_double(float(sd_a)))

    def sample(self, f):
        f, fp = po._f64(np.asarray(f, np.float64).ravel())
        lib().accel_slam_sample(self._g, fp)

    def result(self):
        a = np.zeros(3)
        st = lib().accel_slam_result(self._g, po._p(a, f64p))
        return a, int(st)

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
        n = self.n
        x = np.zeros(n)
        P = np.zeros((n, n), order="F")
        lib().cons_slam_get_state(self.h, po._p(x, f64p), po._p(P, f64p))
        return x, P

    def step(self, frame):
        frame, fp = po._u8(frame)
        lib().accel_slam_step(self._g, fp)

    def features(self):
        nf = self.num_features
        out = dict(label=np.zeros(nf, np.int32), h=np.zeros((nf, 2)), z=np.zeros((nf, 2)),
                   S=np.zeros((nf, 4)), flags=np.zeros(nf, np.uint8),
                   attempted=np.zeros(nf, np.int32), successful=np.zeros(nf, np.int32),
                   select_rank=np.zeros(nf, np.int32))
        lib().cons_slam_get_features(self.h, po._p(out["label"], i32p), po._p(out["h"], f64p),
                                     po._p(out["z"], f64p), po._p(out["S"], f64p), po._p(out["flags"], u8p),
                                     po._p(out["attempted"], i32p), po._p(out["successful"], i32p),
                                     po._p(out["select_rank"], i32p))
        return out


def slam_from_scene(sc, cam8=None, search_override=None, x0=None, P0=None):
    """Slam of a scene (synth.Scene or a rendered scene with cam8, boxsize, y, xp_org, patches, x0, P0)."""
    cam8 = sc.cam8 if cam8 is None else cam8
    so = getattr(sc, "search_override", (0.0, 0.0, 0.0)) if search_override is None else search_override
    n_sel = getattr(sc, "n_select", None) or len(sc.patches)
    cfg = po.make_config(width=int(cam8[0]), height=int(cam8[1]), fku=cam8[2], fkv=cam8[3], u0=cam8[4], v0=cam8[5],
                         kd1=cam8[6], sd=cam8[7], delta_t=getattr(sc, "delta_t", 1.0 / 30.0), n_select=n_sel,
                         boxsize=sc.boxsize, search_override=so)
    s = Slam(cfg)
    x0 = sc.x0 if x0 is None else x0
    for i in range(len(sc.patches)):
        s.add_feature(x0[13 + 3 * i:16 + 3 * i], sc.xp_org[i], sc.patches[i])
    s.set_state(x0, sc.P0 if P0 is None else P0)
    return s
