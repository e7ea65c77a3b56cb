"""GPU parity of the patch search on the adversarial cases of search_cases.py: constructed ties across lanes, strips and
tiles, near-ties across the filter's 1e-5 window, sigma = 10 knife edges, degenerate and huge ellipses.  The filtered
kernel is held to the CPU oracle, to the unfiltered kernel's own score dump, to itself across tile radii from 1 to the
largest the shared memory allows and across batchings, and the SMOE search to the oracle on the same images."""
import numpy as np
import pytest

import search_cases as sc
from gpu_util import ctx_for_image, sl2

pytestmark = pytest.mark.gpu
CAP = 1 << 17       # score_map capacity: a whole 320 x 240 box is ~71 000 candidates


def _ctx(c, radius=20):
    return ctx_for_image(c.image, c.patches, radius=radius)


def _search(ctx, c, jobs, stream=0, slot=0):
    return ctx.patch_search(stream, slot, c.feat[jobs], c.centres[jobs], c.pu[jobs])


def _result_bytes(res):
    return b"".join(np.ascontiguousarray(x).tobytes() for x in res)


def _per_job(res, k):
    return tuple(np.ascontiguousarray(x[k]).tobytes() for x in res)


@pytest.mark.parametrize("B", sc.BOXES)
def test_search_edges_against_oracle(oracle, B):
    """Every job of the box in one call: found flags, positions and the bits of the best score; copy ties go to the
    winner computed from the rules alone."""
    c = sc.cases(B)
    ctx = _ctx(c)
    js = np.arange(len(c.labels))
    u, v, f, best = _search(ctx, c, js)
    ou, ov, of, obest = oracle.elliptical_search(c.image, c.patches[c.feat], c.centres, c.pu)
    bad = [c.labels[j] for j in js
           if f[j] != of[j] or best[j].tobytes() != obest[j].tobytes()
           or (obest[j] < 1e6 and (u[j], v[j]) != (ou[j], ov[j])) or (obest[j] >= 1e6 and (u[j], v[j]) != (-1, -1))]
    assert not bad, bad
    for j, uv in c.winner.items():
        assert (u[j], v[j]) == uv and f[j] == 1, c.labels[j]
    assert f.any() and not f.all()
    ctx.close()


def _dump_argmin(c, j, corr, sd, inside, box):
    """The filtered search's answer from the unfiltered kernel's dump: the least score among candidates inside the
    ellipse, with window and template sigma >= 10 and score <= 1e6; on ties the last scan index."""
    t = c.patches[c.feat[j]].astype(np.int64)
    ok0 = not (sc.sigma_fp64(int(t.sum()), int((t * t).sum()), c.B * c.B) < 10.0)
    ok = (inside.ravel() > 0) & ~(sd.ravel() < 10.0) & (corr.ravel() <= 1e6) & ok0
    if not ok.any():
        return -1, -1, 1e6
    cc = np.where(ok, corr.ravel(), np.inf)
    idx = np.flatnonzero(cc == cc.min())[-1]
    rows = box[3] - box[2] + 1
    return box[4] + box[0] + idx // rows, box[5] + box[2] + idx % rows, cc[idx]


@pytest.mark.parametrize("B", sc.BOXES)
def test_filtered_search_equals_unfiltered_dump(oracle, B):
    """A sample of every family: the unfiltered kernel's every-candidate dump is bit-identical to the oracle's score
    map, and the filtered kernel returns the arg-min taken from that dump."""
    c = sc.cases(B)
    ctx = _ctx(c)
    for j in c.sample(per_family=5) + c.straddle_jobs[::3]:
        box, corr, sd, inside = ctx.score_map(0, 0, c.feat[j], c.centres[j], c.pu[j], cap=CAP)
        obox, ocorr, osd, oinside = oracle.score_map(c.image, c.patches[c.feat[j]], c.centres[j], c.pu[j])
        assert (box == obox).all(), c.labels[j]
        assert inside.tobytes() == oinside.tobytes(), c.labels[j]
        assert corr.tobytes() == ocorr.tobytes() and sd.tobytes() == osd.tobytes(), c.labels[j]
        u, v, f, best = _search(ctx, c, [j])
        du, dv, dbest = _dump_argmin(c, j, corr, sd, inside, box)
        assert (u[0], v[0]) == (du, dv) and best[0] == dbest and f[0] == (dbest <= 0.4), c.labels[j]
    ctx.close()


def test_largest_tile_radius_fits_the_shared_memory():
    import torch
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    for B in sc.BOXES:
        assert sc.largest_radius(B, optin) == sc.SWEEP[-1] == 87, (B, optin)
        c = sc.cases(B)
        with pytest.raises(sl2.Sl2Error):
            _ctx(c, radius=sc.SWEEP[-1] + 1)
        ctx = _ctx(c, radius=sc.SWEEP[-1])       # the context after a refused one works
        _search(ctx, c, [0])
        ctx.close()


@pytest.mark.parametrize("B", sc.BOXES)
def test_tile_radius_sweep_is_bit_identical(B):
    """The tile only changes how the box is walked: every job's result and the sample's score dumps are the same bytes
    at every radius (tiles narrower and shorter than a strip at radius 1 - 3, one tile per box at 87)."""
    c = sc.cases(B)
    js = np.arange(len(c.labels))
    dumps = [j for j in c.sample(per_family=2)]
    ref = None
    for r in (20,) + tuple(x for x in sc.SWEEP if x != 20):
        ctx = _ctx(c, radius=r)
        res = _search(ctx, c, js)
        maps = [ctx.score_map(0, 0, c.feat[j], c.centres[j], c.pu[j], cap=CAP) for j in dumps]
        ctx.close()
        if ref is None:
            ref = (res, maps)
            continue
        diff = [c.labels[j] for j in js if _per_job(res, j) != _per_job(ref[0], j)]
        assert not diff, (r, diff)
        for j, m, m0 in zip(dumps, maps, ref[1]):
            assert all(a.tobytes() == b.tobytes() for a, b in zip(m, m0)), (r, c.labels[j])


@pytest.mark.parametrize("B", sc.BOXES)
def test_batch_independence(B):
    """A job's result does not depend on the other jobs of its call, on their order or on the call's size (1, 3, 4,
    5 and 33 jobs: jobs per stream not a multiple of the 4 warps of a CTA), nor on the stream and ring slot."""
    c = sc.cases(B)
    ctx = _ctx(c)
    js = np.arange(len(c.labels))
    one = _search(ctx, c, js)
    want = [_per_job(one, j) for j in js]
    rev = _search(ctx, c, js[::-1])
    assert [_per_job(rev, k) for k in range(len(js))][::-1] == want
    for size in (1, 3, 4, 5, 33):
        for lo in range(0, len(js), size):
            part = js[lo:lo + size]
            res = _search(ctx, c, part)
            for k, j in enumerate(part):
                assert _per_job(res, k) == want[j], (size, c.labels[j])
    ctx.close()
    # stream 1, slot 1 of a two-stream, two-slot context; the other stream and slot hold a different frame
    cfg = sl2.default_config()
    cfg.width, cfg.height, cfg.boxsize = sc.W, sc.H, B
    cfg.num_streams, cfg.frame_slots = 2, 2
    cfg.max_features = len(c.patches)
    cfg.search_tile_radius = 20
    ctx = sl2.Context(cfg)
    n = len(c.patches)
    other = np.ascontiguousarray(c.image[::-1, ::-1])
    ctx.set_features(0, np.zeros((n, 3)), np.tile([0, 0, 0, 1, 0, 0, 0.0], (n, 1)), c.patches[::-1])
    ctx.set_features(1, np.zeros((n, 3)), np.tile([0, 0, 0, 1, 0, 0, 0.0], (n, 1)), c.patches)
    for s, slot, img in ((0, 0, other), (0, 1, other), (1, 0, other), (1, 1, c.image)):
        ctx.set_frame(s, slot, img)
    res = _search(ctx, c, js, stream=1, slot=1)
    assert _result_bytes(res) == _result_bytes(one)
    ctx.close()


@pytest.mark.parametrize("B", sc.BOXES)
def test_smoe_edges_against_oracle(oracle, B):
    """SMOE search (truncated centres, +5 penalty below sigma 10, shared scores) on the same image and templates: up to
    256 overlapping ellipses per call, clipped at every border, knife-edge windows, the flat corner."""
    c = sc.cases(B)
    ctx = _ctx(c)
    for label, patch, pu, centres in sc.smoe_cases(B):
        ou, ov, of, _ = oracle.smoe_search(c.image, patch, pu, centres)
        ru, rv, rf = ctx.smoe_search_patch(0, 0, patch, pu, centres)
        assert (ru == ou).all() and (rv == ov).all() and (rf == of).all(), label
        f = next(k for k in range(len(c.patches)) if c.patches[k].tobytes() == patch.tobytes())
        ru, rv, rf = ctx.smoe_search(0, 0, f, pu, centres)
        assert (ru == ou).all() and (rv == ov).all() and (rf == of).all(), label
    ctx.close()
