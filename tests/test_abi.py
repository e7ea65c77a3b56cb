"""CPU-side checks of the drop-in boundary: libsl2b200.so loads without a GPU, exports every
symbol include/sl2b200.h declares, and refuses to run without a device (no CPU fallback); the ctypes
mirrors of lib.py lay out every struct and hold every constant as the host C compiler reads the header."""
import collections
import ctypes as C
import os
import re
import subprocess

import pytest

import scenelib2_b200.lib as mirror

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


# One case per C struct that lib.py mirrors: the struct, its ctypes class, its field names in declaration order, the
# size the header fixes for it, a NumPy dtype that mirrors it as well, and {C constant: values it must equal}.
AbiCase = collections.namedtuple("AbiCase", "struct mirror fields size dtype consts", defaults=(None, None, {}))
ABI_CASES = [
    AbiCase("sl2_config", mirror.Sl2Config,
            ("device", "num_streams", "frame_slots", "width", "height", "boxsize", "max_features",
             "number_of_features_to_select", "search_tile_radius", "fku", "fkv", "u0", "v0", "kd1", "sd", "delta_t",
             "search_override", "minimum_attempted_measurements_of_feature", "successful_match_fraction",
             "cuda_stream")),
    AbiCase("sl2_stream_config", mirror.Sl2StreamConfig,
            ("width", "height", "fku", "fkv", "u0", "v0", "kd1", "sd", "delta_t", "number_of_features_to_select")),
    AbiCase("sl2_stream_source", mirror.Sl2StreamSource, ("format", "width", "height", "reserved"),
            consts={"SL2_SRC_GRAY_RING": (mirror.SL2_SRC_GRAY_RING,), "SL2_SRC_GRAY8": (mirror.SL2_SRC_GRAY8,),
                    "SL2_SRC_RGB24": (mirror.SL2_SRC_RGB24,), "SL2_SRC_UYVY": (mirror.SL2_SRC_UYVY,),
                    "SL2_MAX_SOURCE_DIM": (mirror.SL2_MAX_SOURCE_DIM,)}),
    AbiCase("sl2_snapshot_header", mirror.Sl2SnapshotHeader,
            ("magic", "version", "header_bytes", "reserved0", "total_bytes", "boxsize", "nfeat", "n", "reserved1",
             "cam", "nsel", "nvisible", "nmeas", "ncull"), size=128,
            consts={"SL2_SNAPSHOT_MAGIC": (mirror.SL2_SNAPSHOT_MAGIC,),
                    "SL2_SNAPSHOT_VERSION": (mirror.SL2_SNAPSHOT_VERSION,)}),
    AbiCase("sl2_snapshot_sections", mirror.Sl2SnapshotSections, ("x", "P", "field", "templates", "total"),
            consts={"SL2_SNAPSHOT_FIELDS": (len(mirror.SNAPSHOT_FIELDS),)}),
    AbiCase("sl2_step_record", mirror.Sl2StepRecord,
            ("step", "nfeat", "nvisible", "nsel", "nmeas", "nculled", "m", "nis", "logdet_s", "xv", "pxx_diag"),
            size=256, dtype=mirror.STEP_RECORD_DTYPE, consts={"SL2_MAX_RECORDS": (mirror.SL2_MAX_RECORDS, 4096)}),
    AbiCase(None, None, (), consts={"SL2_MAX_FEATURES": (mirror.SL2_MAX_FEATURES, 256),
                                    "SL2_MAX_MEASURED": (mirror.SL2_MAX_MEASURED, 128)}),
]


def _c_layout(tmp_path, case):
    """What the host C compiler makes of include/sl2b200.h: {"sizeof": (size,), field: (offset, size),
    constant: (value,)}."""
    st = case.struct
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "sl2b200.h"', "int main(void) {"]
    if st:
        lines.append('  printf("sizeof %%zu\\n", sizeof(%s));' % st)
    lines += ['  printf("%s %%zu %%zu\\n", offsetof(%s, %s), sizeof(((%s *)0)->%s));' % (f, st, f, st, f)
              for f in case.fields]
    lines += ['  printf("%s %%lld\\n", (long long)(%s));' % (c, c) for c in case.consts]
    lines += ["  return 0;", "}"]
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(lines) + "\n")
    subprocess.check_call([os.environ.get("CC", "cc"), "-std=c99", "-I", os.path.join(ROOT, "include"), "-o",
                           str(exe), str(src)])
    return {ln.split()[0]: tuple(int(v) for v in ln.split()[1:])
            for ln in subprocess.check_output([str(exe)], text=True).splitlines()}


@pytest.mark.parametrize("case", ABI_CASES, ids=lambda case: case.struct or "constants")
def test_ctypes_mirror_matches_header(tmp_path, case):
    """sizeof and every field's offset and size of the struct, as the host C compiler lays it out, equal the ctypes
    mirror (and the NumPy dtype where there is one); the header's constants equal lib.py's."""
    out = _c_layout(tmp_path, case)
    for name, values in case.consts.items():
        assert all(out[name] == (v,) for v in values), (name, out[name], values)
    if case.struct is None:
        return
    M = case.mirror
    assert [f for f, _ in M._fields_] == list(case.fields)
    assert out["sizeof"] == (C.sizeof(M),)
    assert case.size is None or C.sizeof(M) == case.size
    for f, t in M._fields_:
        assert out[f] == (getattr(M, f).offset, C.sizeof(t)), f
    if case.dtype is not None:
        assert list(case.dtype.names) == list(case.fields) and case.dtype.itemsize == C.sizeof(M)
        for f in case.fields:
            assert out[f] == (case.dtype.fields[f][1], case.dtype.fields[f][0].itemsize), f
