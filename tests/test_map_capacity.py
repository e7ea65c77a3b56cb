"""Map capacity and measurement capacity of a context, checked without a GPU.

A stream holds up to SL2_MAX_FEATURES = 256 map features (n <= 781); one step measures at most SL2_MAX_MEASURED =
128 of them (m <= 256).  sl2_create validates both before it looks for a device, so the rules hold on any machine.
"""
import pytest


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    import scenelib2_b200 as sl2
    return sl2


def _cfg(lib, max_features, n_select):
    cfg = lib.default_config()
    cfg.max_features = max_features
    cfg.number_of_features_to_select = n_select
    return cfg


def _create_rc(lib, cfg):
    import ctypes as C
    L = lib.load()
    h = C.c_void_p()
    rc = L.sl2_create(C.byref(cfg), C.byref(h))
    if rc == 0:
        L.sl2_destroy(h)
    return rc, L.sl2_last_error(None).decode()


@pytest.mark.parametrize("max_features, n_select, rule", [
    (257, 10, "bad sizes"),                              # above the map capacity
    (0, 10, "bad sizes"),
    (200, 129, "number_of_features_to_select"),          # a large map measures at most 128 features per step
    (256, 256, "number_of_features_to_select"),
])
def test_create_rejects_capacity_beyond_the_limits(lib, max_features, n_select, rule):
    rc, err = _create_rc(lib, _cfg(lib, max_features, n_select))
    assert rc == -1, (rc, err)                           # SL2_ERR_ARG, before any device query
    assert rule in err, err


@pytest.mark.parametrize("max_features, n_select", [
    (256, 128),     # the largest map with the largest selection
    (129, 10),      # the reference's regime on a map just above 128
    (128, 500),     # at or below 128 the selection never exceeds the map: any value stays valid
    (100, 100),
])
def test_create_accepts_capacity_within_the_limits(lib, max_features, n_select):
    """Passes validation; without a GPU creation then fails for want of a device, on an H100 it succeeds."""
    rc, err = _create_rc(lib, _cfg(lib, max_features, n_select))
    if rc != 0:
        assert rc == -2 and "no CPU fallback" in err, (rc, err)    # SL2_ERR_CUDA: no device on this machine
