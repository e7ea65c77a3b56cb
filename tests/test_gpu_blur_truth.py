"""The device's blurred templates (sl2_blur_templates) against the exposure blur from its definition
(tests/blur_truth.py) on every decided byte, over the CPU tests' cases (tests/test_blur.py): every camera, |q| != 1,
rates from rest to beyond the 32-sample cap, offsets, warp on and off, and seeded normals."""
import numpy as np
import pytest

import blur_truth as bt
import scenelib2_b200 as sl2
from test_blur import CASES


def ctx_for_camera(cam8, B, n=1):
    cfg = sl2.default_config()
    cfg.width, cfg.height = int(cam8[0]), int(cam8[1])
    cfg.boxsize = B
    cfg.max_features = n
    cfg.number_of_features_to_select = n
    cfg.fku, cfg.fkv, cfg.u0, cfg.v0, cfg.kd1, cfg.sd = [float(v) for v in cam8[2:8]]
    return sl2.Context(cfg)


@pytest.mark.gpu
def test_device_equals_the_truth_on_every_decided_byte():
    rng = np.random.default_rng(43)
    ctxs = {}
    checked, ks = 0, set()
    try:
        for i, (name, cam8, B, y, xo, x, ex, off, warp, T) in enumerate(CASES):
            key = (np.asarray(cam8).tobytes(), B)
            if key not in ctxs:
                ctxs[key] = ctx_for_camera(cam8, B)
            ctx = ctxs[key]
            theta = tuple(rng.uniform(-0.3, 0.3, 2)) if i % 3 == 2 else (0.0, 0.0)
            ctx.set_features(0, np.asarray(y)[None], np.asarray(xo)[None], np.asarray(T, np.uint8)[None])
            ctx.set_stream_warp(0, int(warp))
            ctx.set_stream_normals(0, 2 if i % 3 == 2 else 0)
            if i % 3 == 2:
                ctx.set_patch_normals(0, [0], np.array([theta]), np.array([[0.1, 0.0, 0.1]]))
            ctx.set_stream_blur(0, 1, ex, off)
            out, valid, K = ctx.blur_templates(0, [0], x)
            t = bt.blur_truth(cam8, T, y, xo, x, ex, off, warp, theta=theta)
            case_ok, mask = bt.decided(t)
            if not case_ok:
                continue
            if t.v is None:
                assert valid[0] != 2, name
                continue
            assert valid[0] == 2 and K[0] == t.K, (name, K, t.K, t.L)
            assert (out[0][mask] == t.byte[mask]).all(), (name, np.argwhere(out[0] != t.byte))
            checked += 1
            ks.add(int(K[0]))
        assert checked >= 0.6 * len(CASES) and 1 in ks and 32 in ks, (checked, ks)
    finally:
        for c in ctxs.values():
            c.close()
