"""TEST INFRASTRUCTURE ONLY.  ctypes binding of tests/subpixel_oracle.cpp: the sub-pixel refinement (include/sl2b200.h,
sl2_set_stream_subpixel) on top of the CPU oracle of oracle/ and the consensus and rescue oracles, which it uses
unchanged.  The library is compiled on first use, with the oracle's flags, into a directory under the system's
temporary directory named after the hash of its sources, so the repository tree is never written."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import pyoracle as po

_HERE = os.path.dirname(os.path.abspath(__file__))
_ORACLE = os.path.join(os.path.dirname(_HERE), "oracle")
_SRC = os.path.join(_HERE, "subpixel_oracle.cpp")
_DEPS = [_SRC, os.path.join(_HERE, "rescue_oracle.cpp"), os.path.join(_HERE, "consensus_oracle.cpp")]

u8p, i32p, f64p = po.u8p, po.i32p, po.f64p
_lib = None


def _build():
    h = hashlib.sha256()
    for p in _DEPS + sorted(os.path.join(_ORACLE, f) for f in os.listdir(_ORACLE) if f.endswith((".hpp", ".h"))):
        h.update(open(p, "rb").read())
    d = os.path.join(tempfile.gettempdir(), "sl2_subpixel_oracle_%d_%s" % (os.getuid(), h.hexdigest()[:16]))
    so = os.path.join(d, "libsubpixel_oracle.so")
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
        L.sub_slam_create.restype = C.c_void_p
        L.sub_slam_base.restype = C.c_void_p
        L.sub_slam_base.argtypes = [C.c_void_p]
        L.sub_refine.restype = C.c_int32
        for name in ("sub_slam_destroy", "sub_slam_set", "sub_slam_step", "sub_slam_refined"):
            getattr(L, name).restype = None
        L.sub_slam_set.argtypes = [C.c_void_p, C.c_double, C.c_double]
        L.cons_slam_num_features.restype = C.c_int32
        L.cons_slam_state_size.restype = C.c_int32
        for name in ("cons_slam_add_feature", "cons_slam_set_state", "cons_slam_get_state", "cons_slam_get_features"):
            getattr(L, name).restype = None
        _lib = L
    return _lib


def refine(image, width, height, patch, u, v):
    """The oracle's refinement of one successful match -> (zu, zv, refined)."""
    image, ip = po._u8(image)
    patch, pp = po._u8(patch)
    z = np.array([float(u), float(v)])
    ok = lib().sub_refine(ip, C.c_int32(width), C.c_int32(height), pp, C.c_int32(patch.shape[0]), C.c_int32(u),
                          C.c_int32(v), po._p(z, f64p))
    return z[0], z[1], bool(ok)


class Slam:
    """The oracle's whole step with the refinement, the consensus (tau) and the rescue (chi2).  features() sets flags
    bit 3 (8) like sl2_get_features."""

    def __init__(self, cfg):
        self._r = C.c_void_p(lib().sub_slam_create(C.byref(cfg)))
        self.h = C.c_void_p(lib().sub_slam_base(self._r))

    def __del__(self):
        if getattr(self, "_r", None):
            lib().sub_slam_destroy(self._r)
            self._r = self.h = None

    def set_consensus(self, tau, chi2=0.0):
        lib().sub_slam_set(self._r, float(tau), float(chi2))

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
        lib().sub_slam_step(self._r, fp)

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
        ref = np.zeros(nf, np.uint8)
        lib().sub_slam_refined(self._r, po._p(ref, u8p))
        out["flags"] |= ref << 3
        return out


def slam_from_scene(sc, tau, chi2):
    """Slam of a synth.Scene (or a scene with the same fields) with the consensus at tau and the rescue at chi2."""
    cfg = po.make_config(width=sc.width, height=sc.height, fku=sc.cam8[2], fkv=sc.cam8[3], u0=sc.cam8[4],
                         v0=sc.cam8[5], kd1=sc.cam8[6], sd=sc.cam8[7], delta_t=sc.delta_t, n_select=sc.n_select,
                         boxsize=sc.boxsize, search_override=sc.search_override)
    s = Slam(cfg)
    for i in range(sc.n_features):
        s.add_feature(sc.x0[13 + 3 * i:16 + 3 * i], sc.xp_org[i], sc.patches[i])
    s.set_state(sc.x0, sc.P0)
    s.set_consensus(tau, chi2)
    return s
