"""CPU-side checks of the drop-in boundary: libsl2b200.so loads without a GPU, exports every
symbol include/sl2b200.h declares, and refuses to run without a device (no CPU fallback)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    import scenelib2_b200 as sl2
    return sl2


def test_header_symbols_exported(lib):
    hdr = open(os.path.join(ROOT, "include", "sl2b200.h")).read()
    declared = sorted(set(re.findall(r"\b(sl2_[a-z_0-9]+)\s*\(", hdr)))
    assert len(declared) >= 25
    L = lib.load()
    for name in declared:
        assert hasattr(L, name), name
    assert sorted(lib.lib.EXPORTS) == declared
    assert b"sm_90a" in L.sl2_version()


def test_config_struct_matches_header_defaults(lib):
    cfg = lib.default_config()
    assert (cfg.width, cfg.height, cfg.boxsize) == (320, 240, 11)        # cfg:24-25, monoslam.cpp:48
    assert cfg.number_of_features_to_select == 10 and abs(cfg.delta_t - 0.033333333) < 1e-15
    assert (cfg.fku, cfg.u0, cfg.v0, cfg.kd1) == (195.0, 162.0, 125.0, 9e-6)
    assert cfg.minimum_attempted_measurements_of_feature == 10 and cfg.successful_match_fraction == 0.5


def test_no_cpu_fallback(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(lib.Sl2Error) as e:
        lib.Context(lib.default_config())
    assert "no CPU fallback" in str(e.value)


def test_product_does_not_touch_oracle():
    """The shipped package must never import, link or execute anything under oracle/."""
    pkg = os.path.join(ROOT, "scenelib2_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h", ".hpp", ".txt", ".cmake")):
                src = open(os.path.join(dirpath, f), errors="ignore").read()
                code = "\n".join(l for l in src.splitlines()
                                 if not l.strip().startswith(("//", "#", "*", '"""')))
                assert "pyoracle" not in code and "liboracle" not in code and "sl2_oracle" not in code, f
