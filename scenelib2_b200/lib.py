"""ctypes binding of libsl2b200.so — the C ABI declared in include/sl2b200.h.

This module is the Python mirror of the reference-facing boundary: the names and argument
meaning follow MonoSLAM / Kalman (see the header for file:line of each replaced interface).
There is NO fallback: if the CUDA library is missing or no sm_90 device is usable, calls raise.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsl2b200.so")

u8p = C.POINTER(C.c_uint8)
i32p = C.POINTER(C.c_int32)
f64p = C.POINTER(C.c_double)
f32p = C.POINTER(C.c_float)

SL2_MAX_FEATURES = 256   # map capacity per stream (n <= 781)
SL2_MAX_MEASURED = 128   # features one step can measure (m <= 256)


class Sl2Config(C.Structure):
    _fields_ = [
        ("device", C.c_int32), ("num_streams", C.c_int32), ("frame_slots", C.c_int32),
        ("width", C.c_int32), ("height", C.c_int32), ("boxsize", C.c_int32),
        ("max_features", C.c_int32), ("number_of_features_to_select", C.c_int32),
        ("search_tile_radius", C.c_int32),
        ("fku", C.c_double), ("fkv", C.c_double), ("u0", C.c_double), ("v0", C.c_double),
        ("kd1", C.c_double), ("sd", C.c_double), ("delta_t", C.c_double),
        ("search_override", C.c_double * 3),
        ("minimum_attempted_measurements_of_feature", C.c_int32),
        ("successful_match_fraction", C.c_double),
        ("cuda_stream", C.c_void_p),
    ]


class Sl2StreamConfig(C.Structure):
    """sl2_stream_config: one camera stream's camera, image size, frame period and selection count."""
    _fields_ = [
        ("width", C.c_int32), ("height", C.c_int32),
        ("fku", C.c_double), ("fkv", C.c_double), ("u0", C.c_double), ("v0", C.c_double),
        ("kd1", C.c_double), ("sd", C.c_double), ("delta_t", C.c_double),
        ("number_of_features_to_select", C.c_int32),
    ]


class Sl2StreamSource(C.Structure):
    """sl2_stream_source: the raw frame format and size a camera stream takes (SL2_SRC_*; 0 x 0 for the default)."""
    _fields_ = [("format", C.c_int32), ("width", C.c_int32), ("height", C.c_int32), ("reserved", C.c_int32)]


class Sl2StreamSelection(C.Structure):
    """sl2_stream_selection: how a camera stream chooses the features it measures (SL2_SELECT_*)."""
    _fields_ = [("mode", C.c_int32), ("reserved", C.c_int32), ("min_bits", C.c_double)]


SL2_SELECT_TRACE, SL2_SELECT_INFORMATION = 0, 1


class Sl2StreamGyro(C.Structure):
    """sl2_stream_gyro: a camera stream's gyroscope: on, the camera-to-gyro rotation R_gc, the bias and the covariance
    of one sample (row-major, gyro frame)."""
    _fields_ = [("on", C.c_int32), ("reserved", C.c_int32), ("R_gc", C.c_double * 9), ("bias", C.c_double * 3),
                ("cov", C.c_double * 9)]

class Sl2StreamAccel(C.Structure):
    """sl2_stream_accel: a camera stream's accelerometer: on, the camera-to-accelerometer rotation R_ac, the bias and
    the covariance of one sample (row-major, accelerometer frame, m/s^2), the world-frame gravity and sd_a."""
    _fields_ = [("on", C.c_int32), ("reserved", C.c_int32), ("R_ac", C.c_double * 9), ("bias", C.c_double * 3),
                ("cov", C.c_double * 9), ("gravity", C.c_double * 3), ("sd_a", C.c_double)]


class Sl2StreamBlur(C.Structure):
    """sl2_stream_blur: a camera stream's exposure blur: on, the exposure (s) and the exposure's middle relative to
    the frame's time (s)."""
    _fields_ = [("on", C.c_int32), ("reserved", C.c_int32), ("exposure", C.c_double), ("offset", C.c_double)]


class Sl2StreamIterated(C.Structure):
    """sl2_stream_iterated: a camera stream's iterated EKF update: relinearisations allowed (0 = off) and the step
    tolerance in prior standard deviations."""
    _fields_ = [("max_iterations", C.c_int32), ("reserved", C.c_int32), ("tol", C.c_double)]


SL2_MAX_ITERATIONS = 8


class Sl2StreamNormals(C.Structure):
    """sl2_stream_normals: a camera stream's patch normal estimation: Gauss-Newton steps per alignment (0 = off), the
    prior sigma of each tilt component of a new feature, the grey-level noise of one pixel and the per-alignment
    random-walk sigma of the tilt."""
    _fields_ = [("max_iterations", C.c_int32), ("reserved", C.c_int32), ("sigma0", C.c_double),
                ("sigma_i", C.c_double), ("sigma_step", C.c_double)]


SL2_MAX_NORMAL_ITERATIONS = 8

SL2_SRC_GRAY_RING, SL2_SRC_GRAY8, SL2_SRC_RGB24, SL2_SRC_UYVY = 0, 1, 2, 3
SL2_MAX_SOURCE_DIM = 4096
SOURCE_BPP = {SL2_SRC_GRAY8: 1, SL2_SRC_RGB24: 3, SL2_SRC_UYVY: 2}


# every symbol include/sl2b200.h declares (checked by tests/test_abi.py)
EXPORTS = [
    "sl2_default_config", "sl2_create", "sl2_destroy", "sl2_last_error", "sl2_sync", "sl2_version",
    "sl2_set_stream_config", "sl2_get_stream_config", "sl2_set_stream_consensus", "sl2_get_stream_consensus",
    "sl2_set_stream_rescue", "sl2_get_stream_rescue",
    "sl2_set_stream_warp", "sl2_get_stream_warp", "sl2_warp_templates",
    "sl2_set_stream_blur", "sl2_get_stream_blur", "sl2_blur_templates",
    "sl2_set_stream_subpixel", "sl2_get_stream_subpixel",
    "sl2_set_stream_selection", "sl2_get_stream_selection",
    "sl2_set_stream_gyro", "sl2_get_stream_gyro", "sl2_set_gyro_samples", "sl2_gyro_update", "sl2_get_gyro_results",
    "sl2_set_stream_accel", "sl2_get_stream_accel", "sl2_set_accel_samples", "sl2_accel_predict",
    "sl2_get_accel_results",
    "sl2_set_stream_iterated", "sl2_get_stream_iterated", "sl2_get_iterated_results",
    "sl2_set_stream_normals", "sl2_get_stream_normals", "sl2_get_patch_normals", "sl2_set_patch_normals",
    "sl2_align_normals",
    "sl2_set_frame", "sl2_set_frames", "sl2_set_frames_dev",
    "sl2_set_stream_source", "sl2_get_stream_source", "sl2_frame_set_layout", "sl2_set_features",
    "sl2_num_features", "sl2_state_size", "sl2_set_state", "sl2_get_state", "sl2_delete_feature", "sl2_append_feature",
    "sl2_patch_search", "sl2_score_map", "sl2_smoe_search", "sl2_find_best_patch", "sl2_ekf_predict",
    "sl2_predict_measurements", "sl2_make_measurements", "sl2_ekf_update",
    "sl2_ekf_update_measured", "sl2_normalise_state", "sl2_step", "sl2_step_host",
    "sl2_step_host_async", "sl2_wait_slot", "sl2_set_step_groups", "sl2_join", "sl2_measure_particles", "sl2_measure_particles_patch",
    "sl2_smoe_search_patch", "sl2_measure_partial_features",
    "sl2_get_features", "sl2_get_feature_jacobians", "sl2_enable_timing", "sl2_last_step_times", "sl2_last_update_times", "sl2_launch_count",
    "sl2_snapshot_layout", "sl2_snapshot_bytes", "sl2_save_streams", "sl2_load_streams", "sl2_save_streams_dev", "sl2_load_streams_dev",
    "sl2_enable_records", "sl2_get_records", "sl2_get_records_dev", "sl2_relocalise",
    "sl2_set_stream_recovery", "sl2_get_stream_recovery", "sl2_get_recovery_results",
]

SL2_RELOC_HYPOTHESES = 1024   # three-point hypotheses per stream and sl2_relocalise call
SL2_RELOC_GN_ITERS = 5        # Gauss-Newton steps of the refinement


class Sl2RelocParams(C.Structure):
    """sl2_reloc_params: inlier radius, acceptance count and the velocity state of a relocalisation."""
    _fields_ = [("inlier_px", C.c_double), ("min_inliers", C.c_int32), ("reserved", C.c_int32),
                ("v", C.c_double * 3), ("omega", C.c_double * 3)]


class Sl2RelocResult(C.Structure):
    """sl2_reloc_result: what sl2_relocalise found for one stream."""
    _fields_ = [("status", C.c_int32), ("matches", C.c_int32), ("support", C.c_int32), ("inliers", C.c_int32),
                ("rms_px", C.c_double), ("pose", C.c_double * 7)]


# the same result as a NumPy structured dtype: Context.relocalise returns an array of it
RELOC_RESULT_DTYPE = np.dtype([("status", np.int32), ("matches", np.int32), ("support", np.int32),
                               ("inliers", np.int32), ("rms_px", np.float64), ("pose", np.float64, (7,))])



class Sl2StreamRecovery(C.Structure):
    """sl2_stream_recovery: a camera stream's loss detector (lost_after = 0: off) and the relocalisation the fused
    step then tries (the parameters and restart covariance of sl2_relocalise)."""
    _fields_ = [("lost_after", C.c_int32), ("min_matches", C.c_int32), ("retry_period", C.c_int32),
                ("reserved", C.c_int32), ("reloc", Sl2RelocParams), ("Pxx", C.c_double * 169)]


class Sl2RecoveryResult(C.Structure):
    """sl2_recovery_result: a camera stream's recovery state after the last step."""
    _fields_ = [("lost", C.c_int32), ("failed_steps", C.c_int32), ("lost_steps", C.c_int32), ("attempted", C.c_int32),
                ("recoveries", C.c_int64), ("last", Sl2RelocResult)]


# the same state as a NumPy structured dtype: Context.recovery_results returns an array of it
RECOVERY_RESULT_DTYPE = np.dtype([("lost", np.int32), ("failed_steps", np.int32), ("lost_steps", np.int32),
                                  ("attempted", np.int32), ("recoveries", np.int64), ("last", RELOC_RESULT_DTYPE)])

SL2_SNAPSHOT_MAGIC = 0x53324C53
SL2_SNAPSHOT_VERSION = 1


class Sl2SnapshotHeader(C.Structure):
    """sl2_snapshot_header: the fixed header of one stream's snapshot blob."""
    _fields_ = [
        ("magic", C.c_uint32), ("version", C.c_uint32), ("header_bytes", C.c_uint32), ("reserved0", C.c_uint32),
        ("total_bytes", C.c_uint64),
        ("boxsize", C.c_int32), ("nfeat", C.c_int32), ("n", C.c_int32), ("reserved1", C.c_int32),
        ("cam", Sl2StreamConfig),
        ("nsel", C.c_int32), ("nvisible", C.c_int32), ("nmeas", C.c_int32), ("ncull", C.c_int32),
    ]


class Sl2SnapshotSections(C.Structure):
    """sl2_snapshot_sections: byte offsets of a blob's sections (what sl2_snapshot_layout returns)."""
    _fields_ = [("x", C.c_uint64), ("P", C.c_uint64), ("field", C.c_uint64 * 15), ("templates", C.c_uint64),
                ("total", C.c_uint64)]


# the per-feature sections of a snapshot in blob order: (name, per-feature shape, dtype)
SNAPSHOT_FIELDS = (
    ("xp_org", (7,), np.float64), ("attempted", (), np.int32), ("successful", (), np.int32),
    ("h", (2,), np.float64), ("S", (4,), np.float64), ("Rvar", (), np.float64), ("dh_dxp", (2, 7), np.float64),
    ("dh_dy", (2, 3), np.float64), ("sel_rank", (), np.int32), ("z_uv", (2,), np.int32), ("found", (), np.uint8),
    ("best", (), np.float64), ("job_feat", (), np.int32), ("job_centre", (2,), np.float64),
    ("job_puinv", (3,), np.float64),
)


def _align8(b):
    return (b + 7) & ~7


def snapshot_layout(nfeat, boxsize):
    """Byte offset of every section of a snapshot of `nfeat` features and the blob's total size (the format of
    include/sl2b200.h): dict name -> (offset, shape, dtype), and total."""
    n = 13 + 3 * nfeat
    out = {}
    o = C.sizeof(Sl2SnapshotHeader)
    for name, shape, dt in (("x", (n,), np.float64), ("P", (n, n), np.float64)) + tuple(
            (nm, (nfeat,) + sh, dt) for nm, sh, dt in SNAPSHOT_FIELDS) + (
            ("templates", (nfeat, boxsize, boxsize), np.uint8),):
        out[name] = (o, shape, dt)
        o += _align8(int(np.prod(shape, dtype=np.int64)) * np.dtype(dt).itemsize)
    return out, o


def read_snapshot(blob):
    """Parse one stream's snapshot blob: a dict with the header fields, the stream config as `cam` (a dict) and every
    section as a NumPy array (P as an n x n array, column-major like sl2_get_state).  Raises ValueError for a blob
    that is not a snapshot of this version, or is shorter than its header says."""
    blob = bytes(blob)
    hsz = C.sizeof(Sl2SnapshotHeader)
    if len(blob) < hsz:
        raise ValueError("snapshot shorter than its header")
    h = Sl2SnapshotHeader.from_buffer_copy(blob[:hsz])
    if h.magic != SL2_SNAPSHOT_MAGIC or h.version != SL2_SNAPSHOT_VERSION or h.header_bytes != hsz:
        raise ValueError("not a version-%d snapshot in this byte order" % SL2_SNAPSHOT_VERSION)
    if h.reserved0 or h.reserved1:
        raise ValueError("reserved snapshot header fields are not 0")
    if h.nfeat < 0 or h.n != 13 + 3 * h.nfeat:
        raise ValueError("bad map size in the snapshot header")
    layout, total = snapshot_layout(h.nfeat, h.boxsize)
    if h.total_bytes != total:
        raise ValueError("snapshot total size %d does not match nfeat and boxsize (%d)" % (h.total_bytes, total))
    if len(blob) < total:
        raise ValueError("truncated snapshot: %d of %d bytes" % (len(blob), total))
    out = {k: getattr(h, k) for k, _ in Sl2SnapshotHeader._fields_ if k not in ("cam", "reserved0", "reserved1")}
    out["cam"] = {k: getattr(h.cam, k) for k, _ in Sl2StreamConfig._fields_}
    for name, (o, shape, dt) in layout.items():
        cnt = int(np.prod(shape, dtype=np.int64))
        a = np.frombuffer(blob, dtype=dt, count=cnt, offset=o)
        out[name] = a.reshape(shape[::-1]).T.copy() if name == "P" else a.reshape(shape).copy()
    return out


SL2_MAX_RECORDS = 4096   # records kept per stream at most (sl2_enable_records)


class Sl2StepRecord(C.Structure):
    """sl2_step_record: one camera stream's record of one fused step (256 bytes)."""
    _fields_ = [
        ("step", C.c_int64), ("nfeat", C.c_int32), ("nvisible", C.c_int32), ("nsel", C.c_int32), ("nmeas", C.c_int32),
        ("nculled", C.c_int32), ("m", C.c_int32), ("nis", C.c_double), ("logdet_s", C.c_double),
        ("xv", C.c_double * 13), ("pxx_diag", C.c_double * 13),
    ]


# the same record as a NumPy structured dtype: Context.records returns arrays of it
STEP_RECORD_DTYPE = np.dtype([
    ("step", np.int64), ("nfeat", np.int32), ("nvisible", np.int32), ("nsel", np.int32), ("nmeas", np.int32),
    ("nculled", np.int32), ("m", np.int32), ("nis", np.float64), ("logdet_s", np.float64),
    ("xv", np.float64, (13,)), ("pxx_diag", np.float64, (13,)),
])

_lib = None


class Sl2Error(RuntimeError):
    pass


def load():
    """dlopen libsl2b200.so; raises if it has not been built (no silent fallback)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise Sl2Error("%s not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(there is no CPU fallback)" % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        L.sl2_last_error.restype = C.c_char_p
        L.sl2_last_error.argtypes = [C.c_void_p]
        L.sl2_version.restype = C.c_char_p
        L.sl2_launch_count.restype = C.c_int64
        L.sl2_launch_count.argtypes = [C.c_void_p]
        L.sl2_destroy.restype = None
        L.sl2_destroy.argtypes = [C.c_void_p]
        L.sl2_default_config.restype = None
        L.sl2_set_stream_config.argtypes = [C.c_void_p, C.c_int32, C.POINTER(Sl2StreamConfig)]
        L.sl2_get_stream_config.argtypes = [C.c_void_p, C.c_int32, C.POINTER(Sl2StreamConfig)]
        L.sl2_set_stream_consensus.argtypes = [C.c_void_p, C.c_int32, C.c_double]
        L.sl2_get_stream_consensus.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_double)]
        L.sl2_set_stream_rescue.argtypes = [C.c_void_p, C.c_int32, C.c_double]
        L.sl2_get_stream_rescue.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_double)]
        L.sl2_set_stream_warp.argtypes = [C.c_void_p, C.c_int32, C.c_int32]
        L.sl2_get_stream_warp.argtypes = [C.c_void_p, C.c_int32, i32p]
        L.sl2_set_stream_blur.argtypes = [C.c_void_p, C.c_int32, C.POINTER(Sl2StreamBlur)]
        L.sl2_get_stream_blur.argtypes = [C.c_void_p, C.c_int32, C.POINTER(Sl2StreamBlur)]
        L.sl2_blur_templates.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_void_p]
        L.sl2_set_stream_subpixel.argtypes = [C.c_void_p, C.c_int32, C.c_int32]
        L.sl2_get_stream_subpixel.argtypes = [C.c_void_p, C.c_int32, i32p]
        L.sl2_set_stream_selection.argtypes = [C.c_void_p, C.c_int32, C.POINTER(Sl2StreamSelection)]
        L.sl2_get_stream_selection.argtypes = [C.c_void_p, C.c_int32, C.POINTER(Sl2StreamSelection)]
        L.sl2_set_stream_gyro.argtypes = [C.c_void_p, C.c_int32, C.POINTER(Sl2StreamGyro)]
        L.sl2_get_stream_gyro.argtypes = [C.c_void_p, C.c_int32, C.POINTER(Sl2StreamGyro)]
        L.sl2_set_gyro_samples.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
        L.sl2_gyro_update.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]
        L.sl2_get_gyro_results.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
        L.sl2_set_stream_accel.argtypes = [C.c_void_p, C.c_int32, C.POINTER(Sl2StreamAccel)]
        L.sl2_get_stream_accel.argtypes = [C.c_void_p, C.c_int32, C.POINTER(Sl2StreamAccel)]
        L.sl2_set_accel_samples.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
        L.sl2_accel_predict.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]
        L.sl2_get_accel_results.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
        L.sl2_set_stream_iterated.argtypes = [C.c_void_p, C.c_int32, C.POINTER(Sl2StreamIterated)]
        L.sl2_get_stream_iterated.argtypes = [C.c_void_p, C.c_int32, C.POINTER(Sl2StreamIterated)]
        L.sl2_get_iterated_results.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
        L.sl2_set_stream_normals.argtypes = [C.c_void_p, C.c_int32, C.POINTER(Sl2StreamNormals)]
        L.sl2_get_stream_normals.argtypes = [C.c_void_p, C.c_int32, C.POINTER(Sl2StreamNormals)]
        L.sl2_get_patch_normals.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_void_p, C.c_void_p]
        L.sl2_set_patch_normals.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
        L.sl2_align_normals.argtypes = [C.c_void_p, C.c_int32, C.c_int32]
        L.sl2_warp_templates.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p]
        L.sl2_set_frame.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_size_t]
        L.sl2_set_frames.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]
        L.sl2_set_frames_dev.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]
        L.sl2_set_stream_source.argtypes = [C.c_void_p, C.c_int32, C.POINTER(Sl2StreamSource)]
        L.sl2_get_stream_source.argtypes = [C.c_void_p, C.c_int32, C.POINTER(Sl2StreamSource)]
        L.sl2_frame_set_layout.argtypes = [C.c_void_p, C.POINTER(C.c_size_t)]
        L.sl2_step.argtypes = [C.c_void_p, C.c_int32]
        L.sl2_step_host.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
        L.sl2_step_host_async.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
        L.sl2_wait_slot.argtypes = [C.c_void_p, C.c_int32]
        L.sl2_set_step_groups.argtypes = [C.c_void_p, C.c_int32]
        L.sl2_join.argtypes = [C.c_void_p]
        L.sl2_measure_particles.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, f64p, f64p,
                                            f64p, f64p, C.c_double, f64p, i32p, u8p, u8p, f64p, f64p]
        L.sl2_measure_particles_patch.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, f64p,
                                                  f64p, f64p, f64p, C.c_double, f64p, i32p, u8p, u8p, f64p, f64p]
        L.sl2_smoe_search_patch.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, f64p, f64p,
                                            i32p, i32p, u8p]
        L.sl2_sync.argtypes = [C.c_void_p]
        L.sl2_score_map.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, f64p, f64p, i32p,
                                    f64p, f64p, u8p, C.c_size_t]
        L.sl2_snapshot_layout.argtypes = [C.c_int32, C.c_int32, C.POINTER(Sl2SnapshotSections)]
        L.sl2_snapshot_bytes.restype = C.c_size_t
        L.sl2_snapshot_bytes.argtypes = [C.c_void_p]
        L.sl2_save_streams.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_size_t,
                                       C.POINTER(C.c_size_t)]
        L.sl2_load_streams.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_size_t]
        L.sl2_save_streams_dev.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_size_t]
        L.sl2_load_streams_dev.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_size_t]
        L.sl2_enable_records.argtypes = [C.c_void_p, C.c_int32]
        L.sl2_get_records.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
        L.sl2_get_records_dev.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
        L.sl2_relocalise.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.POINTER(Sl2RelocParams),
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.sl2_set_stream_recovery.argtypes = [C.c_void_p, C.c_int32, C.POINTER(Sl2StreamRecovery)]
        L.sl2_get_stream_recovery.argtypes = [C.c_void_p, C.c_int32, C.POINTER(Sl2StreamRecovery)]
        L.sl2_get_recovery_results.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]
        _lib = L
    return _lib


def default_config():
    cfg = Sl2Config()
    load().sl2_default_config(C.byref(cfg))
    return cfg


def _p(a, t):
    return a.ctypes.data_as(t)


def _f64(a):
    a = np.ascontiguousarray(a, dtype=np.float64)
    return a, _p(a, f64p)


def _colmajor(a):
    a = np.asfortranarray(np.asarray(a, np.float64))
    return a, _p(a, f64p)


class Context:
    """One GPU context holding `num_streams` independent camera streams."""

    def __init__(self, cfg):
        self.L = load()
        self.cfg = cfg
        h = C.c_void_p()
        rc = self.L.sl2_create(C.byref(cfg), C.byref(h))
        if rc != 0:
            raise Sl2Error("sl2_create failed (%d): %s" % (rc, self.L.sl2_last_error(None).decode()))
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.L.sl2_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def _ck(self, rc):
        if rc < 0:
            raise Sl2Error("libsl2b200 error %d: %s" % (rc, self.L.sl2_last_error(self.h).decode()))
        return rc

    # ---- per-stream camera ----------------------------------------------------------------------
    def set_stream_config(self, stream_id, sc=None, **fields):
        """sl2_set_stream_config: `sc` (an Sl2StreamConfig, default the stream's current one) with `fields`
        (width, height, fku, fkv, u0, v0, kd1, sd, delta_t, number_of_features_to_select) replaced."""
        if sc is None:
            sc = self.stream_config(stream_id)
        else:
            sc = Sl2StreamConfig.from_buffer_copy(sc)
        for k, v in fields.items():
            if k not in dict(Sl2StreamConfig._fields_):
                raise TypeError("unknown sl2_stream_config field %r" % k)
            setattr(sc, k, v)
        self._ck(self.L.sl2_set_stream_config(self.h, stream_id, C.byref(sc)))

    def stream_config(self, stream_id):
        sc = Sl2StreamConfig()
        self._ck(self.L.sl2_get_stream_config(self.h, stream_id, C.byref(sc)))
        return sc

    # ---- match consensus ----------------------------------------------------------------------
    def set_stream_consensus(self, stream_id, inlier_px):
        """sl2_set_stream_consensus: reject the step's matches that disagree with the best one-point hypothesis by
        more than inlier_px pixels before the EKF update (0 = off, the default)."""
        self._ck(self.L.sl2_set_stream_consensus(self.h, stream_id, float(inlier_px)))

    def stream_consensus(self, stream_id):
        v = C.c_double()
        self._ck(self.L.sl2_get_stream_consensus(self.h, stream_id, C.byref(v)))
        return v.value

    def set_stream_rescue(self, stream_id, chi2):
        """sl2_set_stream_rescue: after the update with the consensus's inliers, take back the rejected matches whose
        innovation at the updated state has nu^T S^-1 nu <= chi2, and update with them (0 = off, the default; 5.991
        is the 95 % point of chi^2 with two degrees of freedom)."""
        self._ck(self.L.sl2_set_stream_rescue(self.h, stream_id, float(chi2)))

    def stream_rescue(self, stream_id):
        v = C.c_double()
        self._ck(self.L.sl2_get_stream_rescue(self.h, stream_id, C.byref(v)))
        return v.value

    # ---- feature selection ----------------------------------------------------------------------
    def set_stream_selection(self, stream_id, mode, min_bits=0.0, reserved=0):
        """sl2_set_stream_selection: choose the stream's measured features by trace (SL2_SELECT_TRACE, the default)
        or greedily by mutual information (SL2_SELECT_INFORMATION), each pick adding more than min_bits bits."""
        sel = Sl2StreamSelection(int(mode), int(reserved), float(min_bits))
        self._ck(self.L.sl2_set_stream_selection(self.h, stream_id, C.byref(sel)))

    def get_stream_selection(self, stream_id):
        """-> (mode, min_bits)"""
        sel = Sl2StreamSelection()
        self._ck(self.L.sl2_get_stream_selection(self.h, stream_id, C.byref(sel)))
        return sel.mode, sel.min_bits

    # ---- planar patch warp ----------------------------------------------------------------------
    def set_stream_warp(self, stream_id, on):
        """sl2_set_stream_warp: search the stream's selected features with their templates warped to the predicted
        viewpoint (1) or with the stored templates (0, the default)."""
        self._ck(self.L.sl2_set_stream_warp(self.h, stream_id, int(on)))

    def get_stream_warp(self, stream_id):
        v = C.c_int32()
        self._ck(self.L.sl2_get_stream_warp(self.h, stream_id, C.byref(v)))
        return v.value

    # ---- sub-pixel refinement ---------------------------------------------------------------------
    def set_stream_subpixel(self, stream_id, on):
        """sl2_set_stream_subpixel: refine the stream's matches to the minimum of a quadratic fit of the search's score
        around them (1) or keep the integer matches (0, the default)."""
        self._ck(self.L.sl2_set_stream_subpixel(self.h, stream_id, int(on)))

    def get_stream_subpixel(self, stream_id):
        v = C.c_int32()
        self._ck(self.L.sl2_get_stream_subpixel(self.h, stream_id, C.byref(v)))
        return v.value

    def warp_templates(self, stream_id, feat_index, xp):
        """sl2_warp_templates: the templates of the features feat_index warped to the camera pose xp (7: r, q), as the
        search of a warp-on stream sees them -> (templates (n, B, B) u8, valid (n,) u8; 0 = the stored template)."""
        feat_index = np.ascontiguousarray(feat_index, np.int32).reshape(-1)
        xp = np.ascontiguousarray(xp, np.float64).reshape(-1)
        if xp.size != 7:
            raise ValueError("xp must hold 7 values (r, q)")
        n, B = feat_index.size, self.cfg.boxsize
        out = np.zeros((n, B, B), np.uint8)
        valid = np.zeros(n, np.uint8)
        self._ck(self.L.sl2_warp_templates(self.h, stream_id, n, feat_index.ctypes.data, xp.ctypes.data,
                                           out.ctypes.data, valid.ctypes.data))
        return out, valid

    # ---- exposure blur ------------------------------------------------------------------------
    def set_stream_blur(self, stream_id, on, exposure=0.0, offset=0.0, reserved=0):
        """sl2_set_stream_blur: search the stream's selected features with their templates blurred along the predicted
        motion over the exposure (seconds; offset = the exposure's middle relative to the frame's time) (on = 1), or
        not (0, the default)."""
        b = Sl2StreamBlur()
        b.on, b.reserved, b.exposure, b.offset = int(on), int(reserved), float(exposure), float(offset)
        self._ck(self.L.sl2_set_stream_blur(self.h, stream_id, C.byref(b)))

    def stream_blur(self, stream_id):
        """-> dict(on, exposure, offset)"""
        b = Sl2StreamBlur()
        self._ck(self.L.sl2_get_stream_blur(self.h, stream_id, C.byref(b)))
        return dict(on=b.on, exposure=b.exposure, offset=b.offset)

    def blur_templates(self, stream_id, feat_index, xv):
        """sl2_blur_templates: the templates the fused search of the stream uses for the features feat_index at the
        state xv (13: r, q, v, omega), with the stream's blur, warp and normals settings -> (templates (n, B, B) u8,
        valid (n,) u8: 0 stored, 1 warped, 2 blurred, samples (n,) i32: K of a blurred template, else 0)."""
        feat_index = np.ascontiguousarray(feat_index, np.int32).reshape(-1)
        xv = np.ascontiguousarray(xv, np.float64).reshape(-1)
        if xv.size < 13:
            raise ValueError("xv must hold 13 values (r, q, v, omega)")
        xv = np.ascontiguousarray(xv[:13])
        n, B = feat_index.size, self.cfg.boxsize
        out = np.zeros((n, B, B), np.uint8)
        valid = np.zeros(n, np.uint8)
        samples = np.zeros(n, np.int32)
        self._ck(self.L.sl2_blur_templates(self.h, stream_id, n, feat_index.ctypes.data, xv.ctypes.data,
                                           out.ctypes.data, valid.ctypes.data, samples.ctypes.data))
        return out, valid, samples

    # ---- gyroscope ----------------------------------------------------------------------------
    def set_stream_gyro(self, stream_id, on, R_gc=None, bias=None, cov=None, reserved=0):
        """sl2_set_stream_gyro: update the stream's omega with one gyroscope sample per step, between the motion
        prediction and the feature prediction (on = 1), or not (0, the default).  R_gc (3x3) takes camera-frame vectors
        into the gyro's frame (default I), bias (3) is in rad/s (default 0), cov (3x3) is the covariance of one sample,
        the mean rate over the frame period (default I)."""
        g = Sl2StreamGyro()
        g.on, g.reserved = int(on), int(reserved)
        for name, v, dflt in (("R_gc", R_gc, np.eye(3)), ("bias", bias, np.zeros(3)), ("cov", cov, np.eye(3))):
            a = np.asarray(dflt if v is None else v, np.float64).reshape(-1)
            if a.size != len(getattr(g, name)):
                raise ValueError("%s must hold %d values" % (name, len(getattr(g, name))))
            getattr(g, name)[:] = [float(t) for t in a]
        self._ck(self.L.sl2_set_stream_gyro(self.h, stream_id, C.byref(g)))

    def stream_gyro(self, stream_id):
        """-> dict(on, R_gc (3x3), bias (3), cov (3x3))"""
        g = Sl2StreamGyro()
        self._ck(self.L.sl2_get_stream_gyro(self.h, stream_id, C.byref(g)))
        return dict(on=g.on, R_gc=np.array(g.R_gc).reshape(3, 3), bias=np.array(g.bias),
                    cov=np.array(g.cov).reshape(3, 3))

    def set_gyro_samples(self, slot, rates, valid=None, lo=0):
        """sl2_set_gyro_samples: the samples (cnt x 3 rad/s, gyro frame) of streams [lo, lo + cnt) for the fused step
        of ring slot `slot`; valid (cnt, None = all) marks the streams that have one."""
        rates = np.ascontiguousarray(rates, np.float64).reshape(-1, 3)
        cnt = rates.shape[0]
        if valid is not None:
            valid = np.ascontiguousarray(valid, np.uint8).reshape(-1)
            if valid.size != cnt:
                raise ValueError("valid must hold one byte per sample")
        self._ck(self.L.sl2_set_gyro_samples(self.h, slot, lo, cnt, rates.ctypes.data,
                                             None if valid is None else valid.ctypes.data))

    def gyro_update(self, stream_id, rate3):
        """sl2_gyro_update: the staged gyro update of one stream with one sample, between ekf_predict and
        predict_measurements."""
        rate3 = np.ascontiguousarray(rate3, np.float64).reshape(-1)
        if rate3.size != 3:
            raise ValueError("rate3 must hold 3 values")
        self._ck(self.L.sl2_gyro_update(self.h, stream_id, rate3.ctypes.data))

    def gyro_results(self, lo=0, cnt=None):
        """sl2_get_gyro_results -> (nis (cnt,), status (cnt,): 0 none this step, 1 applied, 2 skipped)."""
        if cnt is None:
            cnt = self.cfg.num_streams - lo
        nis, status = np.zeros(max(cnt, 0)), np.zeros(max(cnt, 0), np.int32)
        self._ck(self.L.sl2_get_gyro_results(self.h, lo, cnt, nis.ctypes.data, status.ctypes.data))
        return nis, status

    # ---- accelerometer ------------------------------------------------------------------------
    def set_stream_accel(self, stream_id, on, R_ac=None, bias=None, cov=None, gravity=None, sd_a=4.0, reserved=0):
        """sl2_set_stream_accel: drive the stream's motion prediction with one accelerometer sample per step (on = 1),
        or not (0, the default).  R_ac (3x3) takes camera-frame vectors into the accelerometer's frame (default I),
        bias (3) is in m/s^2 (default 0), cov (3x3) is the covariance of one sample, the mean specific force over the
        frame period (default I), gravity (3) is the world-frame gravity vector in m/s^2 (default 0) and sd_a (m/s^2)
        the acceleration a sample does not explain."""
        a = Sl2StreamAccel()
        a.on, a.reserved, a.sd_a = int(on), int(reserved), float(sd_a)
        for name, v, dflt in (("R_ac", R_ac, np.eye(3)), ("bias", bias, np.zeros(3)), ("cov", cov, np.eye(3)),
                              ("gravity", gravity, np.zeros(3))):
            t = np.asarray(dflt if v is None else v, np.float64).reshape(-1)
            if t.size != len(getattr(a, name)):
                raise ValueError("%s must hold %d values" % (name, len(getattr(a, name))))
            getattr(a, name)[:] = [float(u) for u in t]
        self._ck(self.L.sl2_set_stream_accel(self.h, stream_id, C.byref(a)))

    def stream_accel(self, stream_id):
        """-> dict(on, R_ac (3x3), bias (3), cov (3x3), gravity (3), sd_a)"""
        a = Sl2StreamAccel()
        self._ck(self.L.sl2_get_stream_accel(self.h, stream_id, C.byref(a)))
        return dict(on=a.on, R_ac=np.array(a.R_ac).reshape(3, 3), bias=np.array(a.bias),
                    cov=np.array(a.cov).reshape(3, 3), gravity=np.array(a.gravity), sd_a=a.sd_a)

    def set_accel_samples(self, slot, forces, valid=None, lo=0):
        """sl2_set_accel_samples: the samples (cnt x 3 m/s^2, accelerometer frame) of streams [lo, lo + cnt) for the
        fused step of ring slot `slot`; valid (cnt, None = all) marks the streams that have one."""
        forces = np.ascontiguousarray(forces, np.float64).reshape(-1, 3)
        cnt = forces.shape[0]
        if valid is not None:
            valid = np.ascontiguousarray(valid, np.uint8).reshape(-1)
            if valid.size != cnt:
                raise ValueError("valid must hold one byte per sample")
        self._ck(self.L.sl2_set_accel_samples(self.h, slot, lo, cnt, forces.ctypes.data,
                                              None if valid is None else valid.ctypes.data))

    def accel_predict(self, stream_id, f3):
        """sl2_accel_predict: the staged motion prediction of one stream with one accelerometer sample, in place of
        ekf_predict."""
        f3 = np.ascontiguousarray(f3, np.float64).reshape(-1)
        if f3.size != 3:
            raise ValueError("f3 must hold 3 values")
        self._ck(self.L.sl2_accel_predict(self.h, stream_id, f3.ctypes.data))

    def accel_results(self, lo=0, cnt=None):
        """sl2_get_accel_results -> (a (cnt, 3) world-frame m/s^2, status (cnt,): 0 none this step, 1 applied,
        2 skipped)."""
        if cnt is None:
            cnt = self.cfg.num_streams - lo
        a, status = np.zeros((max(cnt, 0), 3)), np.zeros(max(cnt, 0), np.int32)
        self._ck(self.L.sl2_get_accel_results(self.h, lo, cnt, a.ctypes.data, status.ctypes.data))
        return a, status

    # ---- iterated update -----------------------------------------------------------------------
    def set_stream_iterated(self, stream_id, max_iterations, tol=0.0, reserved=0):
        """sl2_set_stream_iterated: relinearise the stream's EKF update at the updated state up to max_iterations
        times (0 = off, the default), stopping once a step moves no state entry by more than tol prior standard
        deviations."""
        v = Sl2StreamIterated(int(max_iterations), int(reserved), float(tol))
        self._ck(self.L.sl2_set_stream_iterated(self.h, stream_id, C.byref(v)))

    def stream_iterated(self, stream_id):
        """-> (max_iterations, tol)"""
        v = Sl2StreamIterated()
        self._ck(self.L.sl2_get_stream_iterated(self.h, stream_id, C.byref(v)))
        return v.max_iterations, v.tol

    def iterated_results(self, lo=0, cnt=None):
        """sl2_get_iterated_results -> (iterations (cnt,), status (cnt,): 0 off or nothing measured, 1 converged,
        2 ran out, 3 invalid relinearisation, last_delta (cnt,))."""
        if cnt is None:
            cnt = self.cfg.num_streams - lo
        k = max(cnt, 0)
        it, st, dl = np.zeros(k, np.int32), np.zeros(k, np.int32), np.zeros(k)
        self._ck(self.L.sl2_get_iterated_results(self.h, lo, cnt, it.ctypes.data, st.ctypes.data, dl.ctypes.data))
        return it, st, dl

    # ---- patch normals -------------------------------------------------------------------------
    def set_stream_normals(self, stream_id, max_iterations, sigma0=0.5, sigma_i=8.0, sigma_step=0.0, reserved=0):
        """sl2_set_stream_normals: estimate each feature's patch normal from the images with up to max_iterations
        Gauss-Newton steps per alignment (0 = off, the default), and warp the stream's templates through it; resets
        the stream's estimates."""
        v = Sl2StreamNormals(int(max_iterations), int(reserved), float(sigma0), float(sigma_i), float(sigma_step))
        self._ck(self.L.sl2_set_stream_normals(self.h, stream_id, C.byref(v)))

    def stream_normals(self, stream_id):
        """-> dict(max_iterations, sigma0, sigma_i, sigma_step)"""
        v = Sl2StreamNormals()
        self._ck(self.L.sl2_get_stream_normals(self.h, stream_id, C.byref(v)))
        return dict(max_iterations=v.max_iterations, sigma0=v.sigma0, sigma_i=v.sigma_i, sigma_step=v.sigma_step)

    def patch_normals(self, stream_id, feat_index):
        """sl2_get_patch_normals -> dict(theta (n, 2), cov (n, 3): S_aa, S_ab, S_bb, normal_w (n, 3) unit world
        normals, count (n,) accepted alignments, status (n,): 0 not aligned, 1 accepted, 2 no step accepted,
        3 invalid start)."""
        feat_index = np.ascontiguousarray(feat_index, np.int32).reshape(-1)
        n = feat_index.size
        th, cv, nw = np.zeros((n, 2)), np.zeros((n, 3)), np.zeros((n, 3))
        ct, st = np.zeros(n, np.int32), np.zeros(n, np.uint8)
        self._ck(self.L.sl2_get_patch_normals(self.h, stream_id, n, feat_index.ctypes.data, th.ctypes.data,
                                              cv.ctypes.data, nw.ctypes.data, ct.ctypes.data, st.ctypes.data))
        return dict(theta=th, cov=cv, normal_w=nw, count=ct, status=st)

    def set_patch_normals(self, stream_id, feat_index, theta, cov):
        """sl2_set_patch_normals: the estimates theta (n, 2) and cov (n, 3: S_aa, S_ab, S_bb) of the features
        feat_index, with count and status 0."""
        feat_index = np.ascontiguousarray(feat_index, np.int32).reshape(-1)
        n = feat_index.size
        theta = np.ascontiguousarray(theta, np.float64).reshape(n, 2)
        cov = np.ascontiguousarray(cov, np.float64).reshape(n, 3)
        self._ck(self.L.sl2_set_patch_normals(self.h, stream_id, n, feat_index.ctypes.data, theta.ctypes.data,
                                              cov.ctypes.data))

    def align_normals(self, stream_id, slot):
        """sl2_align_normals: the stream's normal alignment on ring slot `slot`, as the fused step runs it after its
        update."""
        self._ck(self.L.sl2_align_normals(self.h, stream_id, slot))

    # ---- frames -------------------------------------------------------------------------------
    def set_stream_source(self, stream_id, format, width=0, height=0):
        """sl2_set_stream_source: the stream takes raw `format` frames of width x height (SL2_SRC_*), converted to
        gray and resized to its image on the device; SL2_SRC_GRAY_RING with 0 x 0 restores the default."""
        src = Sl2StreamSource(format, width, height, 0)
        self._ck(self.L.sl2_set_stream_source(self.h, stream_id, C.byref(src)))
        self._sources = None

    def stream_source(self, stream_id):
        src = Sl2StreamSource()
        self._ck(self.L.sl2_get_stream_source(self.h, stream_id, C.byref(src)))
        return src

    def frame_set_layout(self):
        """Byte offsets of the streams' frames in a frame set, and the total (num_streams + 1 entries)."""
        out = (C.c_size_t * (self.cfg.num_streams + 1))()
        self._ck(self.L.sl2_frame_set_layout(self.h, out))
        return [int(v) for v in out]

    def _has_sources(self):
        if getattr(self, "_sources", None) is None:
            self._sources = any(self.stream_source(s).format for s in range(self.cfg.num_streams))
        return self._sources

    def set_frame(self, stream_id, slot, gray):
        """One stream's image (H_s, W_s) or, with a source, its raw frame (height, width[, bpp])."""
        gray = np.ascontiguousarray(gray, np.uint8)
        self._ck(self.L.sl2_set_frame(self.h, stream_id, slot, gray.ctypes.data, gray.strides[0]))
        self._ck(self.L.sl2_sync(self.h))

    def set_frames(self, slot, gray):
        """gray: (num_streams, H, W) u8 host array, or, when a stream has a source, the packed frame set of
        frame_set_layout() (any u8 array of that many bytes)."""
        gray = np.ascontiguousarray(gray, np.uint8)
        if self._has_sources():
            assert gray.nbytes == self.frame_set_layout()[-1]
        else:
            assert gray.shape == (self.cfg.num_streams, self.cfg.height, self.cfg.width)
        self._ck(self.L.sl2_set_frames(self.h, slot, gray.ctypes.data))
        self._ck(self.L.sl2_sync(self.h))

    def set_frames_ptr(self, slot, host_ptr):
        self._ck(self.L.sl2_set_frames(self.h, slot, host_ptr))

    def set_frames_dev(self, slot, dev_ptr):
        self._ck(self.L.sl2_set_frames_dev(self.h, slot, dev_ptr))

    # ---- map / state --------------------------------------------------------------------------
    def set_features(self, stream_id, y, xp_org, patches):
        y, yp = _f64(y)
        xp_org, xp = _f64(xp_org)
        patches = np.ascontiguousarray(patches, np.uint8)
        n = patches.shape[0]
        self._ck(self.L.sl2_set_features(self.h, stream_id, n, yp, xp, _p(patches, u8p)))

    def num_features(self, stream_id):
        return self._ck(self.L.sl2_num_features(self.h, stream_id))

    def state_size(self, stream_id):
        return self._ck(self.L.sl2_state_size(self.h, stream_id))

    def set_state(self, stream_id, x, P):
        x, xp = _f64(x)
        P, pp = _colmajor(P)
        self._ck(self.L.sl2_set_state(self.h, stream_id, xp, pp))

    def get_state(self, stream_id):
        n = self.state_size(stream_id)
        x = np.zeros(n)
        P = np.zeros((n, n), order="F")
        self._ck(self.L.sl2_get_state(self.h, stream_id, _p(x, f64p), _p(P, f64p)))
        return x, P

    def append_feature(self, stream_id, y, xp_org, patch, Pcol=None):
        """MonoSLAM::AddNewKnownFeature on the device; Pcol (n+3, 3) column block or None (zeros). Returns the index."""
        y, yp = _f64(y)
        xp, xpp = _f64(xp_org)
        patch = np.ascontiguousarray(patch, np.uint8)
        pc = None
        if Pcol is not None:
            Pcol = np.asfortranarray(Pcol, dtype=np.float64)   # column-major (n + 3) x 3
            pc = Pcol.ctypes.data_as(f64p)
        return self._ck(self.L.sl2_append_feature(self.h, stream_id, yp, xpp, _p(patch, u8p), pc))

    def delete_feature(self, stream_id, index):
        self._ck(self.L.sl2_delete_feature(self.h, stream_id, index))

    # ---- patch search -------------------------------------------------------------------------
    def patch_search(self, stream_id, slot, feat_index, centres, puinv3):
        feat_index = np.ascontiguousarray(feat_index, np.int32)
        centres, cp = _f64(centres)
        puinv3, qp = _f64(puinv3)
        n = feat_index.size
        u = np.zeros(n, np.int32)
        v = np.zeros(n, np.int32)
        found = np.zeros(n, np.uint8)
        best = np.zeros(n, np.float64)
        self._ck(self.L.sl2_patch_search(self.h, stream_id, slot, n, _p(feat_index, i32p), cp, qp,
                                         _p(u, i32p), _p(v, i32p), _p(found, u8p), _p(best, f64p)))
        return u, v, found, best

    def score_map(self, stream_id, slot, feat_index, centre, puinv3, cap=1 << 16):
        centre, cp = _f64(centre)
        puinv3, qp = _f64(puinv3)
        box = np.zeros(6, np.int32)
        corr = np.zeros(cap)
        sd = np.zeros(cap)
        inside = np.zeros(cap, np.uint8)
        self._ck(self.L.sl2_score_map(self.h, stream_id, slot, feat_index, cp, qp, _p(box, i32p),
                                      _p(corr, f64p), _p(sd, f64p), _p(inside, u8p), cap))
        nu, nv = max(0, box[1] - box[0] + 1), max(0, box[3] - box[2] + 1)
        k = nu * nv
        return box, corr[:k].reshape(nu, nv), sd[:k].reshape(nu, nv), inside[:k].reshape(nu, nv)

    def smoe_search(self, stream_id, slot, feat_index, puinv3, centres):
        puinv3, qp = _f64(puinv3)
        centres, cp = _f64(centres)
        K = puinv3.shape[0]
        ru = np.zeros(K, np.int32)
        rv = np.zeros(K, np.int32)
        rf = np.zeros(K, np.uint8)
        self._ck(self.L.sl2_smoe_search(self.h, stream_id, slot, feat_index, K, qp, cp,
                                        _p(ru, i32p), _p(rv, i32p), _p(rf, u8p)))
        return ru, rv, rf

    def smoe_search_patch(self, stream_id, slot, patch, puinv3, centres):
        """SMOE search with a raw template (not a map feature)."""
        patch = np.ascontiguousarray(patch, np.uint8)
        assert patch.shape == (self.cfg.boxsize, self.cfg.boxsize)
        puinv3, qp = _f64(puinv3)
        centres, cp = _f64(centres)
        K = puinv3.shape[0]
        ru, rv, rf = np.zeros(K, np.int32), np.zeros(K, np.int32), np.zeros(K, np.uint8)
        self._ck(self.L.sl2_smoe_search_patch(self.h, stream_id, slot, patch.ctypes.data, K, qp, cp, _p(ru, i32p),
                                              _p(rv, i32p), _p(rf, u8p)))
        return ru, rv, rf

    def measure_particles(self, stream_id, slot, feat_index, h, Sinv3, detS, lam, prune_threshold, prob,
                          patch=None):
        """N2: SMOE search + particle re-weighting of one partially-initialised feature ->
        survivors, prob, z_uv (K,2), found, keep, cumulative, (mean, variance).  With `patch` (B x B u8) the
        template is given directly instead of naming map feature `feat_index`."""
        h, hp = _f64(h)
        Sinv3, sp = _f64(Sinv3)
        detS, dp = _f64(detS)
        lam, lp = _f64(lam)
        prob = np.array(prob, np.float64)
        K = prob.shape[0]
        z = np.zeros((K, 2), np.int32)
        found = np.zeros(K, np.uint8)
        keep = np.zeros(K, np.uint8)
        cum = np.zeros(K)
        mv = np.zeros(2)
        args = (K, hp, sp, dp, lp, float(prune_threshold), _p(prob, f64p), _p(z, i32p), _p(found, u8p),
                _p(keep, u8p), _p(cum, f64p), _p(mv, f64p))
        if patch is None:
            left = self._ck(self.L.sl2_measure_particles(self.h, stream_id, slot, feat_index, *args))
        else:
            patch = np.ascontiguousarray(patch, np.uint8)
            assert patch.shape == (self.cfg.boxsize, self.cfg.boxsize)
            left = self._ck(self.L.sl2_measure_particles_patch(self.h, stream_id, slot, patch.ctypes.data, *args))
        return left, prob, z, found, keep, cum, mv

    def measure_partial_features(self, stream_id, slot, patches, ypi, Pxy, Pyy, lam, prune_threshold, prob, K=None,
                                 out=None):
        """N2 for F partially-initialised features in one call: device prediction of every particle's ellipse
        (monoslam.cpp:1347-1400), SMOE search with one score map per feature, particle re-weighting.
        patches (F,B,B) u8; ypi (F,6); Pxy (F,13,6); Pyy (F,6,6); lam, prob (F,Kmax); K (F,) particle counts
        (default Kmax).  Returns a dict of arrays; `out` may supply any of them (same shape and dtype), which the call
        then writes in place (slots k >= K[f] keep what they held)."""
        patches = np.ascontiguousarray(patches, np.uint8)
        F = patches.shape[0]
        ypi = np.ascontiguousarray(ypi, np.float64).reshape(F, 6)
        Pxy = np.ascontiguousarray(np.asarray(Pxy, np.float64).reshape(F, 13, 6).transpose(0, 2, 1))  # column-major
        Pyy = np.ascontiguousarray(np.asarray(Pyy, np.float64).reshape(F, 6, 6).transpose(0, 2, 1))
        lam = np.ascontiguousarray(lam, np.float64).reshape(F, -1)
        Kmax = lam.shape[1]
        prob = np.array(prob, np.float64).reshape(F, Kmax)
        K = np.full(F, Kmax, np.int32) if K is None else np.ascontiguousarray(K, np.int32)
        given = out or {}
        out = {"h": np.zeros((F, Kmax, 2)), "Sinv3": np.zeros((F, Kmax, 3)), "detS": np.zeros((F, Kmax)),
               "z": np.zeros((F, Kmax, 2), np.int32), "found": np.zeros((F, Kmax), np.uint8),
               "keep": np.zeros((F, Kmax), np.uint8), "cumulative": np.zeros((F, Kmax)),
               "mean_var": np.zeros((F, 2)), "left": np.zeros(F, np.int32)}
        for k, a in given.items():
            if k not in out or a.shape != out[k].shape or a.dtype != out[k].dtype or not a.flags.c_contiguous:
                raise ValueError("out[%r]: expected a C-contiguous %s array of shape %s" % (k, out[k].dtype,
                                                                                        out[k].shape))
            out[k] = a
        self._ck(self.L.sl2_measure_partial_features(
            self.h, stream_id, slot, F, Kmax, _p(K, i32p), C.c_void_p(patches.ctypes.data), _p(ypi, f64p), _p(Pxy, f64p),
            _p(Pyy, f64p), _p(lam, f64p), C.c_double(float(prune_threshold)), _p(prob, f64p), _p(out["h"], f64p),
            _p(out["Sinv3"], f64p), _p(out["detS"], f64p), _p(out["z"], i32p), _p(out["found"], u8p),
            _p(out["keep"], u8p), _p(out["cumulative"], f64p), _p(out["mean_var"], f64p), _p(out["left"], i32p)))
        out["prob"] = prob
        return out

    def find_best_patch(self, stream_id, slot, regions, ubest=-1, vbest=-1):
        """regions (n,4) = (ustart, vstart, ufinish, vfinish) -> u, v (kept at ubest/vbest where the
        reference would not write them), ev."""
        regions = np.ascontiguousarray(regions, np.int32).reshape(-1, 4)
        n = regions.shape[0]
        u = np.full(n, ubest, np.int32)
        v = np.full(n, vbest, np.int32)
        ev = np.zeros(n, np.float64)
        self._ck(self.L.sl2_find_best_patch(self.h, stream_id, slot, n, _p(regions, i32p), _p(u, i32p),
                                            _p(v, i32p), _p(ev, f64p)))
        return u, v, ev

    # ---- EKF ----------------------------------------------------------------------------------
    def ekf_predict(self, stream_id, u3=None):
        if u3 is None:
            self._ck(self.L.sl2_ekf_predict(self.h, stream_id, None))
        else:
            u3, up = _f64(u3)
            self._ck(self.L.sl2_ekf_predict(self.h, stream_id, up))

    def predict_measurements(self, stream_id):
        return self._ck(self.L.sl2_predict_measurements(self.h, stream_id))

    def make_measurements(self, stream_id, slot):
        return self._ck(self.L.sl2_make_measurements(self.h, stream_id, slot))

    def ekf_update(self, stream_id, feat_index, H_xv, H_y, R, nu):
        """H_xv (m,13), H_y (m,3) row-major; R (m/2, 2, 2); nu (m,)."""
        feat_index = np.ascontiguousarray(feat_index, np.int32)
        H_xv, a = _f64(H_xv)
        H_y, b = _f64(H_y)
        R, r = _f64(R)
        nu, nn = _f64(nu)
        self._ck(self.L.sl2_ekf_update(self.h, stream_id, nu.size, _p(feat_index, i32p), a, b, r, nn))

    def ekf_update_measured(self, stream_id):
        self._ck(self.L.sl2_ekf_update_measured(self.h, stream_id))

    def normalise_state(self, stream_id):
        self._ck(self.L.sl2_normalise_state(self.h, stream_id))

    # ---- fused step ---------------------------------------------------------------------------
    def step(self, slot=0):
        self._ck(self.L.sl2_step(self.h, slot))

    def step_host(self, slot, gray_ptr, xv_out_ptr):
        self._ck(self.L.sl2_step_host(self.h, slot, gray_ptr, xv_out_ptr))

    def step_host_async(self, slot, gray_ptr, xv_out_ptr):
        self._ck(self.L.sl2_step_host_async(self.h, slot, gray_ptr, xv_out_ptr))

    def wait_slot(self, slot):
        self._ck(self.L.sl2_wait_slot(self.h, slot))

    def set_step_groups(self, groups):
        self._ck(self.L.sl2_set_step_groups(self.h, groups))

    def join(self):
        self._ck(self.L.sl2_join(self.h))

    def sync(self):
        self._ck(self.L.sl2_sync(self.h))

    def enable_timing(self, on=True):
        self._ck(self.L.sl2_enable_timing(self.h, 1 if on else 0))

    def last_step_times(self):
        ms = np.zeros(4, np.float32)
        self._ck(self.L.sl2_last_step_times(self.h, _p(ms, f32p)))
        return ms

    def last_update_times(self):
        """ms of the five EKF update kernels of the last step: hp, chol, solve, syrk, finish"""
        ms = np.zeros(5, np.float32)
        self._ck(self.L.sl2_last_update_times(self.h, _p(ms, f32p)))
        return ms

    def launch_count(self):
        return int(self.L.sl2_launch_count(self.h))

    def feature_jacobians(self, stream_id):
        """Feature::dh_by_dxv_ (nf,26), dh_by_dy_ (nf,6), R_ (nf,4), nu_ (nf,2), column-major like the Eigen members"""
        N = self.cfg.max_features
        J, Jy, R, nu = np.zeros((N, 26)), np.zeros((N, 6)), np.zeros((N, 4)), np.zeros((N, 2))
        nf = self._ck(self.L.sl2_get_feature_jacobians(self.h, stream_id, _p(J, f64p), _p(Jy, f64p), _p(R, f64p),
                                                       _p(nu, f64p)))
        return J[:nf], Jy[:nf], R[:nf], nu[:nf]

    def features(self, stream_id):
        N = self.cfg.max_features
        out = dict(h=np.zeros((N, 2)), z=np.zeros((N, 2)), S=np.zeros((N, 4)),
                   flags=np.zeros(N, np.uint8), attempted=np.zeros(N, np.int32),
                   successful=np.zeros(N, np.int32), select_rank=np.zeros(N, np.int32))
        nf = self._ck(self.L.sl2_get_features(
            self.h, stream_id, _p(out["h"], f64p), _p(out["z"], f64p), _p(out["S"], f64p),
            _p(out["flags"], u8p), _p(out["attempted"], i32p), _p(out["successful"], i32p),
            _p(out["select_rank"], i32p)))
        return {k: v[:nf] for k, v in out.items()}

    # ---- stream snapshots -----------------------------------------------------------------------
    def snapshot_bytes(self):
        """Upper bound of one stream's snapshot in this context (a map of max_features features)."""
        return int(self.L.sl2_snapshot_bytes(self.h))

    def save_streams(self, lo=0, cnt=None):
        """Snapshots of the streams [lo, lo + cnt) (default: to the last stream) as a list of bytes."""
        if cnt is None:
            cnt = self.cfg.num_streams - lo
        stride = self.snapshot_bytes()
        buf = np.empty(max(cnt, 0) * stride, np.uint8)
        sizes = (C.c_size_t * max(cnt, 1))()
        self._ck(self.L.sl2_save_streams(self.h, lo, cnt, buf.ctypes.data, stride, sizes))
        return [buf[i * stride:i * stride + sizes[i]].tobytes() for i in range(cnt)]

    def save_stream(self, stream_id):
        return self.save_streams(stream_id, 1)[0]

    def load_streams(self, blobs, lo=0):
        """Load blobs[i] into stream lo + i (all or nothing: on an error no stream changes)."""
        blobs = [bytes(b) for b in blobs]
        stride = _align8(max([len(b) for b in blobs] + [C.sizeof(Sl2SnapshotHeader)]))
        buf = np.zeros(len(blobs) * stride, np.uint8)
        for i, b in enumerate(blobs):
            buf[i * stride:i * stride + len(b)] = np.frombuffer(b, np.uint8)
        self._ck(self.L.sl2_load_streams(self.h, lo, len(blobs), buf.ctypes.data, stride))

    def load_stream(self, stream_id, blob):
        self.load_streams([blob], stream_id)

    def save_streams_dev(self, lo, cnt, dev_ptr, stride):
        """Snapshots of [lo, lo + cnt) into device memory at dev_ptr + i * stride, asynchronous on the context's
        stream (stride >= snapshot_bytes(), both multiples of 8)."""
        self._ck(self.L.sl2_save_streams_dev(self.h, lo, cnt, dev_ptr, stride))

    def load_streams_dev(self, lo, cnt, dev_ptr, stride):
        self._ck(self.L.sl2_load_streams_dev(self.h, lo, cnt, dev_ptr, stride))

    # ---- step records ---------------------------------------------------------------------------
    def enable_records(self, depth):
        """sl2_enable_records: keep the last `depth` step records of every stream (0 = off); restarts `step` at 0."""
        self._ck(self.L.sl2_enable_records(self.h, depth))
        self._rec_depth = depth

    def records(self, lo=0, cnt=None, max=None):
        """The most recent step records of the streams [lo, lo + cnt) (default: to the last stream), oldest first, as a
        structured array of STEP_RECORD_DTYPE of shape [cnt, k], k = min(max, steps recorded, depth); max defaults to
        the depth."""
        if cnt is None:
            cnt = self.cfg.num_streams - lo
        if max is None:
            max = getattr(self, "_rec_depth", 0) or 1
        out = np.zeros((cnt if cnt > 0 else 0, max if max > 0 else 0), STEP_RECORD_DTYPE)  # bad sizes: refused by the C call
        k = self._ck(self.L.sl2_get_records(self.h, lo, cnt, max, out.ctypes.data))
        return out[:, :k]

    def records_dev(self, lo, cnt, max, dev_ptr):
        """sl2_get_records_dev: the same records into device memory at dev_ptr (record i * max + j, 8-byte aligned),
        asynchronous on the context's stream.  Returns k."""
        return self._ck(self.L.sl2_get_records_dev(self.h, lo, cnt, max, dev_ptr))

    # ---- relocalisation -------------------------------------------------------------------------
    def relocalise(self, stream_ids, slot, inlier_px, min_inliers, v, omega, Pxx, reserved=0):
        """sl2_relocalise: search every map feature of each listed stream over its whole frame in `slot`, estimate
        the camera pose with a three-point consensus and, when at least min_inliers matches agree with the refined
        pose, restart the stream's filter there (x[7:13] = v, omega; Pxx; the camera-map correlations zero).
        Returns (results, z_uv, flags): a RELOC_RESULT_DTYPE array (cnt,), int32 (cnt, max_features, 2) and uint8
        (cnt, max_features) (bit0 matched, bit1 inlier of the refined pose)."""
        ids = np.ascontiguousarray(stream_ids, np.int32).reshape(-1)
        cnt = ids.size
        prm = Sl2RelocParams()
        prm.inlier_px, prm.min_inliers, prm.reserved = float(inlier_px), int(min_inliers), int(reserved)
        for i in range(3):
            prm.v[i], prm.omega[i] = float(v[i]), float(omega[i])
        Pxx = np.asfortranarray(np.asarray(Pxx, np.float64).reshape(13, 13))
        N = self.cfg.max_features
        res = np.zeros(max(cnt, 1), RELOC_RESULT_DTYPE)
        z = np.zeros((max(cnt, 1), N, 2), np.int32)
        fl = np.zeros((max(cnt, 1), N), np.uint8)
        self._ck(self.L.sl2_relocalise(self.h, ids.ctypes.data, cnt, slot, C.byref(prm), Pxx.ctypes.data,
                                       res.ctypes.data, z.ctypes.data, fl.ctypes.data))
        return res[:cnt], z[:cnt], fl[:cnt]

    # ---- stream recovery ------------------------------------------------------------------------
    def set_stream_recovery(self, stream_id, lost_after, min_matches=1, retry_period=1, inlier_px=2.0, min_inliers=6,
                            v=(0.0, 0.0, 0.0), omega=(0.0, 0.0, 1e-3), Pxx=None, reserved=0):
        """sl2_set_stream_recovery: after lost_after consecutive steps with fewer than min_matches successful
        measurements (0 = off, the default), the fused step stops the stream's selection and tries sl2_relocalise on
        its frame with these parameters: on the step that declares it lost, then every retry_period-th step."""
        r = Sl2StreamRecovery()
        r.lost_after, r.min_matches, r.retry_period, r.reserved = (int(lost_after), int(min_matches),
                                                                   int(retry_period), int(reserved))
        r.reloc.inlier_px, r.reloc.min_inliers = float(inlier_px), int(min_inliers)
        for i in range(3):
            r.reloc.v[i], r.reloc.omega[i] = float(v[i]), float(omega[i])
        if Pxx is not None:
            P = np.asarray(Pxx, np.float64).reshape(13, 13).flatten(order="F")
            for i in range(169):
                r.Pxx[i] = float(P[i])
        self._ck(self.L.sl2_set_stream_recovery(self.h, stream_id, C.byref(r)))

    def stream_recovery(self, stream_id):
        """-> the stream's Sl2StreamRecovery"""
        r = Sl2StreamRecovery()
        self._ck(self.L.sl2_get_stream_recovery(self.h, stream_id, C.byref(r)))
        return r

    def recovery_results(self, lo=0, cnt=None):
        """sl2_get_recovery_results -> a RECOVERY_RESULT_DTYPE array (cnt,)"""
        if cnt is None:
            cnt = self.cfg.num_streams - lo
        out = np.zeros(max(cnt, 1), RECOVERY_RESULT_DTYPE)
        self._ck(self.L.sl2_get_recovery_results(self.h, lo, cnt, out.ctypes.data))
        return out[:max(cnt, 0)]


def config_for_scene(sc, num_streams=1, frame_slots=1, device=0, max_features=None,
                     cuda_stream=None, search_tile_radius=None):
    """sl2_config matching a synth.Scene."""
    cfg = default_config()
    cfg.device = device
    cfg.num_streams = num_streams
    cfg.frame_slots = frame_slots
    cfg.width, cfg.height = sc.width, sc.height
    cfg.boxsize = sc.boxsize
    cfg.max_features = max_features or sc.n_features
    cfg.number_of_features_to_select = sc.n_select
    if search_tile_radius is None:
        rad = sc.meta.get("config", {}).get("radius") or 20
        search_tile_radius = rad
    cfg.search_tile_radius = search_tile_radius
    cfg.fku, cfg.fkv, cfg.u0, cfg.v0, cfg.kd1, cfg.sd = [float(v) for v in sc.cam8[2:8]]
    cfg.delta_t = sc.delta_t
    for i in range(3):
        cfg.search_override[i] = sc.search_override[i]
    if cuda_stream is not None:
        cfg.cuda_stream = cuda_stream
    return cfg


def stream_config_for_scene(sc):
    """sl2_stream_config matching a synth.Scene's camera, frame period and selection count."""
    out = Sl2StreamConfig()
    out.width, out.height = sc.width, sc.height
    out.fku, out.fkv, out.u0, out.v0, out.kd1, out.sd = [float(v) for v in sc.cam8[2:8]]
    out.delta_t = sc.delta_t
    out.number_of_features_to_select = sc.n_select
    return out


def load_scene(ctx, stream_id, sc):
    """Install a synth.Scene (map + prior) into one stream of a context."""
    n = sc.n_features
    ctx.set_features(stream_id, sc.x0[13:].reshape(n, 3), sc.xp_org, sc.patches)
    ctx.set_state(stream_id, sc.x0, sc.P0)
