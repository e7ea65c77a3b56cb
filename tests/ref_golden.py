"""What the reference's own code returned, stored under tests/golden/ref_<test>.npz, so that the tests that compare
with the original SceneLib2 sources run without them.

The reference side of such a test goes through a Reference object instead of calling oracle/_ref directly.  Replayed
(the default), every call checks a fingerprint of its inputs against the stored one (the test still builds the same
inputs; a relative tolerance of 1e-9 lets through the last-bit differences a machine's BLAS can make in synthetic
inputs such as a covariance built by a matrix product) and returns the stored outputs, in call order.  With SL2_RECORD_REFERENCE=1 and oracle/_ref built from the original
sources (`make -C oracle REF=<SceneLib2 checkout>`), the calls run the live reference and the file is rewritten.

A covariance matrix returned by RefSlam.get_state is stored as its diagonal plus a fixed, seeded sample of
P_SAMPLE entries (the full matrices of a step-by-step run would not fit a repository); the other entries replay as
NaN, and whether the matrix was exactly symmetric is stored with it.
"""
import json
import os

import numpy as np

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
P_SAMPLE = 128
RECORD = os.environ.get("SL2_RECORD_REFERENCE") == "1"


def _fingerprint(args):
    """Size, weighted sum and absolute sum of all numeric arguments (work directories and the like are skipped)."""
    a = [np.asarray(x, np.float64).ravel() for x in args if not isinstance(x, (str, bytes))]
    a = np.concatenate(a) if a else np.zeros(0)
    w = np.sin(np.arange(a.size) * 0.7 + 0.3)
    return np.array([a.size, (a * w).sum(), np.abs(a).sum()])


def _pack(out, store):
    """Structure of `out` as JSON; its arrays are appended to store["f"] (floating point) / store["i"] (integers)."""
    if isinstance(out, dict):
        return {"d": {k: _pack(v, store) for k, v in out.items()}}
    if isinstance(out, (tuple, list)):
        return {"t": [_pack(v, store) for v in out]}
    if out is None:
        return {"n": 0}
    a = np.asarray(out)
    kind = "f" if a.dtype.kind == "f" else "i"
    off = sum(x.size for x in store[kind])
    store[kind].append(a.ravel())
    return {"a": [kind, off, list(a.shape), a.dtype.str], "s": np.isscalar(out) or isinstance(out, (bool, int, float))}


def _unpack(spec, flat):
    if "d" in spec:
        return {k: _unpack(v, flat) for k, v in spec["d"].items()}
    if "t" in spec:
        return tuple(_unpack(v, flat) for v in spec["t"])
    if "n" in spec:
        return None
    kind, off, shape, dtype = spec["a"]
    a = flat[kind][off:off + int(np.prod(shape))].astype(dtype).reshape(shape)
    return a[()] if spec["s"] else a


class Reference:
    """Calls of the reference (live or replayed) for one test."""

    def __init__(self, name, oracle):
        self.path = os.path.join(G, "ref_%s.npz" % name)
        self.oracle = oracle
        self.n = 0
        self.rec = {"f": [], "i": [], "in": []}
        self.rec_specs = []
        if RECORD:
            assert oracle.ref() is not None and oracle.ref_models() is not None, \
                "SL2_RECORD_REFERENCE=1 needs oracle/_ref built from the reference sources"
        else:
            z = np.load(self.path)
            self.flat = {"f": z["f"], "i": z["i"]}
            self.inputs = z["inputs"]
            self.specs = json.loads(str(z["specs"]))

    def call(self, fn, *args, live=None, **kw):
        """Output of the reference function `fn` of oracle/pyoracle (use_ref=True unless `live` is given)."""
        d = _fingerprint(list(args) + [v for v in kw.values()])
        i = self.n
        self.n += 1
        if RECORD:
            out = live(*args, **kw) if live else getattr(self.oracle, fn)(*args, use_ref=True, **kw)
            self.rec["in"].append(d)
            self.rec_specs.append([fn, _pack(out, self.rec)])
            return out
        assert self.specs[i][0] == fn, (i, fn, self.specs[i][0])
        assert np.allclose(self.inputs[i], d, rtol=1e-9, atol=1e-12 * abs(d[2])), \
            "inputs of reference call %d (%s) differ from the recording" % (i, fn)
        return _unpack(self.specs[i][1], self.flat)

    def slam(self, sc, workdir):
        return RefSlam(self, sc, workdir)

    def close(self):
        if RECORD:
            cat = lambda xs, t: np.concatenate(xs).astype(t) if xs else np.zeros(0, t)
            np.savez_compressed(self.path, f=cat(self.rec["f"], np.float64), i=cat(self.rec["i"], np.int64),
                                inputs=np.array(self.rec["in"], np.float64).reshape(-1, 3),
                                specs=np.array(json.dumps(self.rec_specs, separators=(",", ":"))))
        else:
            assert self.n == len(self.specs), "the test made %d of %d recorded reference calls" % (self.n, len(self.specs))


def _sample_P(P, seed):
    n = P.shape[0]
    rng = np.random.default_rng(seed)
    idx = rng.integers(0, n, (P_SAMPLE, 2)).astype(np.int32)
    return dict(diag=np.diag(P).copy(), idx=idx, val=P[idx[:, 0], idx[:, 1]].copy(),
                symmetric=np.array(np.abs(P - P.T).max() == 0.0))


class RefSlam:
    """oracle.RefSlam through a Reference: the same surface; get_state returns P with NaN outside the sample."""

    def __init__(self, ref, sc, workdir):
        self.ref = ref
        self.live = ref.oracle.RefSlam(sc, workdir) if RECORD else None
        ref.call("RefSlam", sc.x0, sc.P0, sc.patches, live=lambda *a: None)

    def _call(self, name, *args, post=None):
        def live(*a):
            out = getattr(self.live, name)
            out = out(*a) if callable(out) else out    # num_features and n are properties
            return post(out) if post else out
        return self.ref.call("RefSlam." + name, *args, live=live)

    @property
    def num_features(self):
        return int(self._call("num_features", post=lambda v: v))

    @property
    def n(self):
        return int(self._call("n", post=lambda v: v))

    def step(self, frame):
        self._call("step", frame)

    def set_state(self, x, P):
        # a replayed P is incomplete: only the call order is checked
        self.ref.call("RefSlam.set_state", live=lambda: self.live.set_state(x, P))

    def init_partial_feature(self, frame, u, v):
        self._call("init_partial_feature", frame, u, v)

    def particle_cycle(self, frame, cap=256):
        return self._call("particle_cycle", frame, cap)

    def features(self):
        return self._call("features")

    def get_state(self):
        seed = self.ref.n
        x, s = self._call("get_state", post=lambda xP: (xP[0], _sample_P(xP[1], seed)))
        self.symmetric = bool(s["symmetric"])
        if RECORD:
            return x, self.live.get_state()[1]
        P = np.full((x.size, x.size), np.nan)
        P[s["idx"][:, 0], s["idx"][:, 1]] = s["val"]
        P[np.arange(x.size), np.arange(x.size)] = s["diag"]
        return x, P
