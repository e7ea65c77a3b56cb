// accel.cu — the accelerometer's entry points: a measured linear acceleration drives the motion prediction of
// predict_kernel (ekf.cu: accel_model, motion_model).  Semantics and the order of every operation: include/sl2b200.h,
// sl2_set_stream_accel; tests/accel_ref.py restates the prediction op for op.  The work runs inside the prediction
// kernel's existing launch: this file holds the setting, the sample ring, the staged form and the results.
#include <algorithm>
#include <cmath>

#include "sl2_context.cuh"

using namespace sl2;

namespace {

// the setting's checks of include/sl2b200.h; an empty string when it is accepted
std::string accel_setting_error(const sl2_stream_accel *a) {
  if (a->reserved != 0 || (a->on != 0 && a->on != 1)) return "reserved must be 0 and on 0 or 1";
  if (!finite_all(a->R_ac, 9) || !finite_all(a->bias, 3) || !finite_all(a->cov, 9) || !finite_all(a->gravity, 3) ||
      !finite_all(&a->sd_a, 1))
    return "non-finite value";
  if (!(a->sd_a >= 0.0)) return "sd_a is negative";
  return sensor_frame_error(a->R_ac, a->cov, "R_ac");
}

Sl2AccelParam accel_param(const sl2_stream_accel &a) {
  Sl2AccelParam p;
  sensor_cov_in_camera(a.R_ac, a.cov, p.Rc);
  for (int i = 0; i < 9; ++i) p.R[i] = a.R_ac[i];
  for (int i = 0; i < 3; ++i) p.b[i] = a.bias[i];
  for (int i = 0; i < 3; ++i) p.g[i] = a.gravity[i];
  p.sd2 = a.sd_a * a.sd_a;
  return p;
}

Sl2Accel accel_table(const sl2_ctx *c) {
  Sl2Accel A = {};
  A.on = c->accel_on_dev;
  A.prm = c->accel_prm;
  A.a = c->accel_a;
  A.status = c->accel_status;
  return A;
}

}  // namespace

namespace sl2 {

Sl2Accel accel_args(const sl2_ctx *c, int slot, int lo, int cnt) {
  if (!any_stream(c, lo, cnt, [](const StreamOptions &o) { return o.accel.on != 0; })) return {};
  Sl2Accel A = accel_table(c);
  A.force = c->accel_force + (size_t)slot * c->d.B * 3;
  A.valid = c->accel_valid + (size_t)slot * c->d.B;
  A.sample_lo = 0;
  return A;
}

}  // namespace sl2

extern "C" {

int sl2_set_stream_accel(sl2_ctx *c, int32_t s, const sl2_stream_accel *a) {
  if (bad_stream(c, s) || !a) return fail(c, SL2_ERR_ARG, "sl2_set_stream_accel: bad argument");
  const std::string why = accel_setting_error(a);
  if (!why.empty()) return fail(c, SL2_ERR_ARG, "sl2_set_stream_accel: " + why);
  const Sl2Dev &d = c->d;
  if (a->on && !c->accel_buf) {
    const size_t B = d.B, slots = d.slots;
    const int rc = alloc_sections(c, c->accel_buf,
                                  {{&c->accel_on_dev, B}, {&c->accel_prm, B * sizeof(Sl2AccelParam)},
                                   {&c->accel_force, slots * B * 3 * sizeof(double)}, {&c->accel_valid, slots * B},
                                   {&c->accel_a, B * 3 * sizeof(double)}, {&c->accel_status, B * sizeof(int)}});
    if (rc) return rc;
  }
  const sl2_stream_accel &old = c->opt[s].accel;
  if (c->accel_buf) {  // pageable copies have read their sources when they return; ordered on the stream, no launch
    const Sl2AccelParam p = accel_param(*a);
    const uint8_t on = (uint8_t)a->on;
    CU_TRY(c, cudaMemcpyAsync(c->accel_prm + s, &p, sizeof p, cudaMemcpyHostToDevice, c->stream));
    if (a->on && !old.on)  // turned on: no stale sample
      CU_TRY(c, cudaMemset2DAsync(c->accel_valid + s, d.B, 0, 1, d.slots, c->stream));
    if (a->on != old.on) {  // turned on or off: no stale result
      CU_TRY(c, cudaMemsetAsync(c->accel_a + 3 * (size_t)s, 0, 3 * sizeof(double), c->stream));
      CU_TRY(c, cudaMemsetAsync(c->accel_status + s, 0, sizeof(int), c->stream));
    }
    CU_TRY(c, cudaMemcpyAsync(c->accel_on_dev + s, &on, 1, cudaMemcpyHostToDevice, c->stream));
  }
  c->opt[s].accel = *a;
  return SL2_OK;
}

int sl2_get_stream_accel(sl2_ctx *c, int32_t s, sl2_stream_accel *a) {
  if (bad_stream(c, s) || !a) return fail(c, SL2_ERR_ARG, "sl2_get_stream_accel: bad argument");
  *a = c->opt[s].accel;
  return SL2_OK;
}

int sl2_set_accel_samples(sl2_ctx *c, int32_t slot, int32_t lo, int32_t cnt, const double *forces,
                          const uint8_t *valid) {
  if (bad_range(c, lo, cnt) || bad_slot(c, slot) || (cnt > 0 && !forces))
    return fail(c, SL2_ERR_ARG, "sl2_set_accel_samples: bad argument");
  std::vector<uint8_t> v(cnt);
  for (int i = 0; i < cnt; ++i) {
    v[i] = (uint8_t)(!valid || valid[i] ? 1 : 0);
    if (v[i] && !finite_all(forces + 3 * (size_t)i, 3))
      return fail(c, SL2_ERR_ARG, "sl2_set_accel_samples: a valid sample with a non-finite force");
  }
  if (!c->accel_buf) return fail(c, SL2_ERR_STATE, "sl2_set_accel_samples: no stream has the accelerometer on");
  if (cnt == 0) return SL2_OK;
  const size_t at = (size_t)slot * c->d.B + lo;
  CU_TRY(c, cudaMemcpyAsync(c->accel_force + 3 * at, forces, sizeof(double) * 3 * cnt, cudaMemcpyHostToDevice,
                            c->stream));
  CU_TRY(c, cudaMemcpyAsync(c->accel_valid + at, v.data(), cnt, cudaMemcpyHostToDevice, c->stream));
  return SL2_OK;
}

int sl2_accel_predict(sl2_ctx *c, int32_t s, const double *f3) {
  if (bad_stream(c, s) || !f3 || !finite_all(f3, 3)) return fail(c, SL2_ERR_ARG, "sl2_accel_predict: bad argument");
  if (!c->opt[s].accel.on) return fail(c, SL2_ERR_STATE, "sl2_accel_predict: the stream's accelerometer is off");
  Stage f{STAGE_IN, 24, f3}, v{STAGE_IN, 1};
  return staged_call(c, {&f, &v}, [&] { v.h[0] = 1; }, [&] {
    Sl2Accel A = accel_table(c);
    A.force = f.dev<double>();
    A.valid = v.d;
    A.sample_lo = s;
    CU_TRY(c, sl2_launch_predict(c->d, s, 1, nullptr, 1, 0, nullptr, queue(c), nullptr, A));
    return SL2_OK;
  });
}

int sl2_get_accel_results(sl2_ctx *c, int32_t lo, int32_t cnt, double *accel, int32_t *status) {
  if (bad_range(c, lo, cnt)) return fail(c, SL2_ERR_ARG, "sl2_get_accel_results: bad range");
  return read_results(c, c->accel_buf != nullptr, lo, cnt,
                      {{accel, c->accel_a, 3 * sizeof(double)}, {status, c->accel_status, sizeof(int)}});
}

}  // extern "C"
