"""TEST INFRASTRUCTURE ONLY.  ctypes binding of tests/selection_oracle.cpp: the mutual-information selection
(include/sl2b200.h, sl2_set_stream_selection) on top of the CPU oracle of oracle/, which it uses unchanged.  The library
is compiled on first use, with the oracle's flags, into a directory under the system's temporary directory named after
the hash of its sources, so the repository tree is never written."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import pyoracle as po

_HERE = os.path.dirname(os.path.abspath(__file__))
_ORACLE = os.path.join(os.path.dirname(_HERE), "oracle")
_SRC = os.path.join(_HERE, "selection_oracle.cpp")

u8p, i32p, f64p = po.u8p, po.i32p, po.f64p
_lib = None


def _build():
    h = hashlib.sha256()
    for p in [_SRC] + sorted(os.path.join(_ORACLE, f) for f in os.listdir(_ORACLE) if f.endswith((".hpp", ".h"))):
        h.update(open(p, "rb").read())
    d = os.path.join(tempfile.gettempdir(), "sl2_selection_oracle_%d_%s" % (os.getuid(), h.hexdigest()[:16]))
    so = os.path.join(d, "libselection_oracle.so")
    if not os.path.exists(so):
        os.makedirs(d, exist_ok=True)
        tmp = so + ".%d.tmp" % os.getpid()
        subprocess.check_call([os.environ.get("CXX", "g++"), "-std=c++17", "-O3", "-DNDEBUG", "-ffp-contract=off",
                               "-fPIC", "-shared", "-pthread", "-I", _ORACLE, "-o", tmp, _SRC, "-Wl,-Bsymbolic",
                               "-Wl,--exclude-libs,ALL"])
        os.replace(tmp, so)
    return so


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(_build())
        L.sel_slam_create.restype = C.c_void_p
        for name in ("sel_slam_destroy", "sel_slam_set_mode", "sel_slam_add_feature", "sel_slam_set_state",
                     "sel_slam_get_state", "sel_slam_step", "sel_slam_get_features"):
            getattr(L, name).restype = None
        L.sel_slam_set_mode.argtypes = [C.c_void_p, C.c_int32, C.c_double]
        _lib = L
    return _lib


class Slam:
    """The oracle's whole step (monoslam.cpp:108-180, tracking only) selecting by `mode` (set_selection: SL2_SELECT_*
    and min_bits).  The surface of pyoracle.Slam that the GPU tests use."""

    def __init__(self, cfg):
        self.h = C.c_void_p(lib().sel_slam_create(C.byref(cfg)))

    def __del__(self):
        if getattr(self, "h", None):
            lib().sel_slam_destroy(self.h)
            self.h = None

    def set_selection(self, mode, min_bits=0.0):
        lib().sel_slam_set_mode(self.h, int(mode), 2.0 ** (2.0 * float(min_bits)))

    def add_feature(self, y, xp_org, patch):
        y, a = po._f64(y)
        xp_org, b = po._f64(xp_org)
        patch, c = po._u8(patch)
        lib().sel_slam_add_feature(self.h, a, b, c)

    @property
    def num_features(self):
        return lib().sel_slam_num_features(self.h)

    @property
    def n(self):
        return lib().sel_slam_state_size(self.h)

    def set_state(self, x, P):
        x, a = po._f64(x)
        P, b = po._colmajor(P)
        lib().sel_slam_set_state(self.h, a, b)

    def get_state(self):
        n = self.n
        x = np.zeros(n)
        P = np.zeros((n, n), order="F")
        lib().sel_slam_get_state(self.h, po._p(x, f64p), po._p(P, f64p))
        return x, P

    def step(self, frame):
        frame, fp = po._u8(frame)
        lib().sel_slam_step(self.h, fp)

    def features(self):
        nf = self.num_features
        out = dict(label=np.zeros(nf, np.int32), h=np.zeros((nf, 2)), z=np.zeros((nf, 2)),
                   S=np.zeros((nf, 4)), flags=np.zeros(nf, np.uint8),
                   attempted=np.zeros(nf, np.int32), successful=np.zeros(nf, np.int32),
                   select_rank=np.zeros(nf, np.int32))
        lib().sel_slam_get_features(self.h, po._p(out["label"], i32p), po._p(out["h"], f64p),
                                     po._p(out["z"], f64p), po._p(out["S"], f64p), po._p(out["flags"], u8p),
                                     po._p(out["attempted"], i32p), po._p(out["successful"], i32p),
                                     po._p(out["select_rank"], i32p))
        return out


def slam_from_scene(sc, mode=1, min_bits=0.0):
    """Slam of a synth.Scene (like gpu_util.oracle_slam_from_scene) selecting by `mode` with min_bits."""
    cfg = po.make_config(width=sc.width, height=sc.height, fku=sc.cam8[2], fkv=sc.cam8[3], u0=sc.cam8[4],
                         v0=sc.cam8[5], kd1=sc.cam8[6], sd=sc.cam8[7], delta_t=sc.delta_t, n_select=sc.n_select,
                         boxsize=sc.boxsize, search_override=sc.search_override)
    s = Slam(cfg)
    for i in range(sc.n_features):
        s.add_feature(sc.x0[13 + 3 * i:16 + 3 * i], sc.xp_org[i], sc.patches[i])
    s.set_state(sc.x0, sc.P0)
    s.set_selection(mode, min_bits)
    return s
