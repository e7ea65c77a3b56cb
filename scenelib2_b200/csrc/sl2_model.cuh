// sl2_model.cuh — the device camera and feature models of predict_kernel and particle_predict_kernel (ekf.cu),
// consensus_kernel (consensus.cu), rescue_kernel (rescue.cu), reloc_kernel (reloc.cu), warp_kernel (warp.cu),
// normals_kernel (normals.cu) and iterate_kernel (iterate.cu).  Everything that decides which pixels are searched
// (S_i, S^-1, h_i) or which match is an inlier uses never-fused rd ops in the oracle's evaluation order.
#pragma once
#include "sl2_common.cuh"

namespace {

struct Quat {
  rd w, x, y, z;
};

__device__ Quat quat_mul(const Quat &a, const Quat &b) {
  Quat q;
  q.w = a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z;
  q.x = a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y;
  q.y = a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z;
  q.z = a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x;
  return q;
}

// QuaternionFromAngularVelocity (math_util.cpp:61-80) of the rotation vector av (omega t): the identity for |av| = 0.
// The motion model (ekf.cu) and the exposure blur (warp.cu) both turn q by it.
__device__ __forceinline__ Quat quat_from_angular_velocity(const rd av[3]) {
  const rd angle = rsqrt_(av[0] * av[0] + av[1] * av[1] + av[2] * av[2]);
  Quat q;
  if (angle.v > 0.0) {
    const rd sn(sin((angle / rd(2.0)).v)), cs(cos((angle / rd(2.0)).v));
    const rd s = sn / angle;
    q.x = s * av[0];
    q.y = s * av[1];
    q.z = s * av[2];
    q.w = cs;
  } else {
    q.w = rd(1.0);
  }
  return q;
}

// Eigen::Quaterniond::inverse(): conjugate / squaredNorm, the zero quaternion when the norm is 0
__device__ __forceinline__ Quat quat_inverse(const Quat &q) {
  const rd n2 = q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z;
  Quat r;
  if (n2.v > 0.0) {
    r.w = q.w / n2;
    r.x = (-q.x) / n2;
    r.y = (-q.y) / n2;
    r.z = (-q.z) / n2;
  }
  return r;
}

// Eigen::Quaterniond::toRotationMatrix()
__device__ __forceinline__ void quat_to_R(const Quat &q, rd R[3][3]) {
  const rd two(2.0), one(1.0);
  const rd tx = two * q.x, ty = two * q.y, tz = two * q.z;
  const rd twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
  const rd txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
  const rd tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
  R[0][0] = one - (tyy + tzz);
  R[0][1] = txy - twz;
  R[0][2] = txz + twy;
  R[1][0] = txy + twz;
  R[1][1] = one - (txx + tzz);
  R[1][2] = tyz - twx;
  R[2][0] = txz - twy;
  R[2][1] = tyz + twx;
  R[2][2] = one - (txx + tyy);
}

// M a, every row summed from 0.0 in ascending order like the oracle
__device__ __forceinline__ void mat3_vec(const rd M[3][3], const rd a[3], rd out[3]) {
  for (int i = 0; i < 3; ++i) {
    rd s(0.0);
    for (int k = 0; k < 3; ++k) s = s + M[i][k] * a[k];
    out[i] = s;
  }
}

// dRq_times_a_by_dq(q, a) (feature_model.cpp:164-185), columns (w, x, y, z): the derivative of the homogeneous form
// R(q) a + (|q|^2 - 1) a, which equals d(R(q) a)/dq along directions tangent to |q| = 1
__device__ __forceinline__ void dRq_times_a_by_dq(const Quat &qi, const rd a[3], rd D[3][4]) {
  const rd two(2.0);
  const rd w2 = two * qi.w, x2 = two * qi.x, y2 = two * qi.y, z2 = two * qi.z;
  const rd m0[9] = {w2, -z2, y2, z2, w2, -x2, -y2, x2, w2};
  const rd mx[9] = {x2, y2, z2, y2, -x2, -w2, z2, w2, -x2};
  const rd my[9] = {-y2, x2, w2, x2, y2, z2, -w2, z2, -y2};
  const rd mz[9] = {-z2, -w2, x2, w2, -z2, y2, x2, y2, z2};
  for (int i = 0; i < 3; ++i) {
    rd s0(0.0), s1(0.0), s2(0.0), s3(0.0);
    for (int k = 0; k < 3; ++k) {
      s0 = s0 + m0[i * 3 + k] * a[k];
      s1 = s1 + mx[i * 3 + k] * a[k];
      s2 = s2 + my[i * 3 + k] * a[k];
      s3 = s3 + mz[i * 3 + k] * a[k];
    }
    D[i][0] = s0;
    D[i][1] = s1;
    D[i][2] = s2;
    D[i][3] = s3;
  }
}
// D dqbar_by_dq (feature_model.cpp:152-162), dqbar_by_dq = diag(1,-1,-1,-1): the derivative by qWR of a term in qRW
__device__ __forceinline__ void times_dqbar_by_dq(rd D[3][4]) {
  for (int i = 0; i < 3; ++i)
    for (int j = 1; j < 4; ++j) D[i][j] = -D[i][j];
}

// RRW of the camera pose xp (position r, quaternion qWR): the rotation of qRW = qWR^-1; returns qRW
__device__ __forceinline__ Quat pose_RRW(const double *xp, rd RRW[3][3]) {
  const Quat qi = quat_inverse(Quat{rd(xp[3]), rd(xp[4]), rd(xp[5]), rd(xp[6])});
  quat_to_R(qi, RRW);
  return qi;
}

// z = RRW (yi - r) with d = yi - r: the camera-frame point of yi seen from xp, RRW = pose_RRW(xp)
__device__ __forceinline__ void zeroed_point(const rd RRW[3][3], const rd yi[3], const double *xp, rd d[3], rd z[3]) {
  for (int i = 0; i < 3; ++i) d[i] = yi[i] - rd(xp[i]);
  mat3_vec(RRW, d, z);
}

// feature_model.cpp:187-238: z = RRW (yi - r), dz/dxp = [-RRW | dRq_times_a_by_dq(qRW, yi - r) dqbar_by_dq]
__device__ __forceinline__ void zeroedyi(const rd yi[3], const double *xp, rd z[3], rd dz_dxp[3][7],
                                         rd RRW[3][3]) {
  rd d[3];
  const Quat qi = pose_RRW(xp, RRW);
  zeroed_point(RRW, yi, xp, d, z);
  rd D[3][4];
  dRq_times_a_by_dq(qi, d, D);
  times_dqbar_by_dq(D);
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) dz_dxp[i][j] = RRW[i][j] * rd(-1.0);
    for (int j = 0; j < 4; ++j) dz_dxp[i][3 + j] = D[i][j];
  }
}

// Camera::Project (camera.cpp:90-114) of the camera-frame point z; uc, vc = the undistorted image-centred point
__device__ __forceinline__ void project_point(const double *cam, const rd z[3], rd h[2], rd &uc, rd &vc) {
  const rd fku(cam[2]), fkv(cam[3]), u0(cam[4]), v0(cam[5]), kd1(cam[6]);
  const rd one(1.0), two(2.0);
  uc = (-fku) * z[0] / z[2];
  vc = (-fkv) * z[1] / z[2];
  const rd radius2 = uc * uc + vc * vc;
  const rd factor = rsqrt_(one + two * kd1 * radius2);
  h[0] = uc / factor + u0;
  h[1] = vc / factor + v0;
}

// Camera::Unproject (camera.cpp:133-157) of the image point h: the camera-frame direction (x, y, 1) that
// project_point maps to h (NaN where 1 - 2 kd1 r^2 < 0, outside the model's reach)
__device__ __forceinline__ void unproject_point(const double *cam, const rd h[2], rd out[3]) {
  const rd fku(cam[2]), fkv(cam[3]), u0(cam[4]), v0(cam[5]), kd1(cam[6]);
  const rd one(1.0), two(2.0);
  const rd c0 = h[0] - u0, c1 = h[1] - v0;
  const rd radius2 = c0 * c0 + c1 * c1;
  const rd factor = rsqrt_(one - two * kd1 * radius2);
  out[0] = (c0 / factor) / (-fku);
  out[1] = (c1 / factor) / (-fkv);
  out[2] = one;
}

// ---- the planar patch warp (include/sl2b200.h, sl2_set_stream_warp; warp_kernel in warp.cu) ------------------------
// a . b, summed from 0.0 in ascending order like mat3_vec
__device__ __forceinline__ rd dot3(const rd a[3], const rd b[3]) {
  rd s(0.0);
  for (int k = 0; k < 3; ++k) s = s + a[k] * b[k];
  return s;
}

// adj(M): A[i][j] = M[j+1][i+1] M[j+2][i+2] - M[j+1][i+2] M[j+2][i+1] (indices mod 3), so that A M = det(M) I
__device__ __forceinline__ void mat3_adj(const rd M[3][3], rd A[3][3]) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      const int j1 = (j + 1) % 3, j2 = (j + 2) % 3, i1 = (i + 1) % 3, i2 = (i + 2) % 3;
      A[i][j] = M[j1][i1] * M[j2][i2] - M[j1][i2] * M[j2][i1];
    }
}

// The patch normal's basis (include/sl2b200.h, sl2_set_stream_normals): nW0 = xo[0:3] - y, E1 = camera o's x axis
// (row 0 of RRWo = pose_RRW(xo)) made orthogonal to nW0 and scaled to |nW0|, E2 = nW0 x E1 / |nW0|
struct PatchBasis {
  rd n0[3], E1[3], E2[3];
};
__device__ __forceinline__ void patch_basis(const double *xo, const rd y[3], const rd RRWo[3][3], PatchBasis &b) {
  for (int i = 0; i < 3; ++i) b.n0[i] = rd(xo[i]) - y[i];
  const rd nn = dot3(b.n0, b.n0);
  const rd pr = dot3(RRWo[0], b.n0) / nn;
  rd q[3];
  for (int i = 0; i < 3; ++i) q[i] = RRWo[0][i] - pr * b.n0[i];
  const rd len = rsqrt_(nn), sc = len / rsqrt_(dot3(q, q));
  for (int i = 0; i < 3; ++i) b.E1[i] = q[i] * sc;
  b.E2[0] = (b.n0[1] * b.E1[2] - b.n0[2] * b.E1[1]) / len;
  b.E2[1] = (b.n0[2] * b.E1[0] - b.n0[0] * b.E1[2]) / len;
  b.E2[2] = (b.n0[0] * b.E1[1] - b.n0[1] * b.E1[0]) / len;
}
// nW(theta) = (nW0 + a E1) + b E2; theta = (0, 0) is nW0 itself
__device__ __forceinline__ void patch_normal(const PatchBasis &b, rd ta, rd tb, rd nW[3]) {
  const bool zero = ta.v == 0.0 && tb.v == 0.0;
  for (int i = 0; i < 3; ++i) nW[i] = zero ? b.n0[i] : (b.n0[i] + ta * b.E1[i]) + tb * b.E2[i];
}

// A camera pose that views a feature's plane (through y, normal nW): adj(RRW) of the pose (the ray's matrix: RRW is a
// rotation only for |q| = 1, quirk Q1, so RRW^T is not its inverse), its position r and num = nW . (y - r)
struct PatchPose {
  rd adj[3][3], r[3], num;
};
// The camera a source position is taken in: its RRW, its position r and the centre c of the template cut there
struct PatchRef {
  rd RRW[3][3], r[3], c[2];
};
// num and r of the pose xp, whose RRW = pose_RRW(xp) and d = y - xp[0:3] (zeroed_point) are given
__device__ __forceinline__ void patch_pose_terms(const double *xp, const rd RRW[3][3], const rd d[3], const rd nW[3],
                                                 PatchPose &p) {
  mat3_adj(RRW, p.adj);
  for (int i = 0; i < 3; ++i) p.r[i] = rd(xp[i]);
  p.num = dot3(nW, d);
}

// What one feature's warp at the camera pose xp shares over its pixels: the feature y seen from xp (h, bit for bit the
// prediction's), the pose xp itself (at), the camera at xo = xp_org with the template centre ho = y seen from xo
// (ref), and the plane through y with normal nW = xo[0:3] - y (nW(theta) when theta, the feature's estimated tilt, is
// given)
struct PatchWarp {
  PatchPose at;
  PatchRef ref;
  rd nW[3];
  rd h[2];
};
__device__ __forceinline__ void patch_warp_setup(const double *cam, const double *xp, const double *xo, const rd y[3],
                                                 PatchWarp &w, const double *theta = nullptr) {
  rd d[3], z[3], uc, vc, RRW[3][3];
  pose_RRW(xp, RRW);
  zeroed_point(RRW, y, xp, d, z);
  project_point(cam, z, w.h, uc, vc);
  rd dox[3], zo[3];
  pose_RRW(xo, w.ref.RRW);
  zeroed_point(w.ref.RRW, y, xo, dox, zo);
  project_point(cam, zo, w.ref.c, uc, vc);
  for (int i = 0; i < 3; ++i) w.ref.r[i] = rd(xo[i]);
  if (theta && (theta[0] != 0.0 || theta[1] != 0.0)) {
    PatchBasis b;
    patch_basis(xo, y, w.ref.RRW, b);
    patch_normal(b, rd(theta[0]), rd(theta[1]), w.nW);
  } else {
    for (int i = 0; i < 3; ++i) w.nW[i] = rd(xo[i]) - y[i];
  }
  patch_pose_terms(xp, RRW, d, w.nW, w.at);
}

// The source position, in the template cut around ref.c in the camera ref, of the ray c (unproject_point of an image
// point) seen from the pose v: dW = adj(RRW) c (= det(RRW) RRW^-1 c, det(RRW) >= 0, and X does not change with the
// scale of dW); t = num / (nW . dW); X = r + t dW; zo = ref.RRW (X - ref.r); src = project_point(zo) - ref.c +
// (half, half).  True when the source is valid: t finite and > 0, zo[2] > 0, src finite.
__device__ __forceinline__ bool patch_ray_source(const double *cam, const PatchPose &v, const PatchRef &ref,
                                                 const rd nW[3], const rd c[3], int half, rd src[2]) {
  rd dW[3];
  mat3_vec(v.adj, c, dW);
  const rd t = v.num / dot3(nW, dW);
  rd e[3], zo[3];
  for (int i = 0; i < 3; ++i) e[i] = (v.r[i] + t * dW[i]) - ref.r[i];
  mat3_vec(ref.RRW, e, zo);
  rd g[2], uc, vc;
  project_point(cam, zo, g, uc, vc);
  src[0] = (g[0] - ref.c[0]) + rd((double)half);
  src[1] = (g[1] - ref.c[1]) + rd((double)half);
  return isfinite(t.v) && t.v > 0.0 && zo[2].v > 0.0 && isfinite(src[0].v) && isfinite(src[1].v);
}

// The warp's source position in the stored template of the output pixel at offset (db, da) (column, row) from the
// centre: patch_ray_source of unproject_point(h + (db, da)) from the pose xp into the camera at xo
__device__ __forceinline__ bool patch_warp_source(const double *cam, const PatchWarp &w, int db, int da, int half,
                                                  rd src[2]) {
  const rd p[2] = {w.h[0] + rd((double)db), w.h[1] + rd((double)da)};
  rd c[3];
  unproject_point(cam, p, c);
  return patch_ray_source(cam, w.at, w.ref, w.nW, c, half, src);
}

// Bilinear value (not rounded) of the box x box template T (row stride ld) at the finite position src (column, row):
// each coordinate clamped to [0, box - 1], so positions outside the template repeat its edge pixels
__device__ __forceinline__ rd patch_bilinear(const uint8_t *T, int ld, int box, const rd src[2]) {
  const double lim = (double)(box - 1);
  const double sx = fmin(fmax(src[0].v, 0.0), lim), sy = fmin(fmax(src[1].v, 0.0), lim);
  const int x0 = min((int)floor(sx), box - 2), y0 = min((int)floor(sy), box - 2);
  const rd fx = rd(sx) - rd((double)x0), fy = rd(sy) - rd((double)y0), one(1.0);
  const uint8_t *r0 = T + y0 * ld + x0, *r1 = r0 + ld;
  const rd top = (one - fx) * rd((double)r0[0]) + fx * rd((double)r0[1]);
  const rd bot = (one - fx) * rd((double)r1[0]) + fx * rd((double)r1[1]);
  return (one - fy) * top + fy * bot;
}
// patch_bilinear rounded to the byte (int)(v + 0.5)
__device__ __forceinline__ int patch_sample(const uint8_t *T, int ld, int box, const rd src[2]) {
  return (int)(patch_bilinear(T, ld, box, src) + rd(0.5)).v;
}

// Camera::Project (camera.cpp:90-114) of the camera-frame point z, and J = dh/dz
// (Camera::ProjectionJacobian, camera.cpp:183-215)
__device__ __forceinline__ void project(const double *cam, const rd z[3], rd h[2], rd J[2][3]) {
  const rd fku(cam[2]), fkv(cam[3]), kd1(cam[6]);
  const rd one(1.0), two(2.0);
  rd uc, vc;
  project_point(cam, z, h, uc, vc);
  const rd fku_yz = fku / z[2], fkv_yz = fkv / z[2];
  rd du[2][3];
  du[0][0] = -fku_yz;
  du[0][1] = rd(0.0);
  du[0][2] = fku_yz * z[0] / z[2];
  du[1][0] = rd(0.0);
  du[1][1] = -fkv_yz;
  du[1][2] = fkv_yz * z[1] / z[2];
  rd dh[2][2];
  dh[0][0] = uc * uc;
  dh[0][1] = uc * vc;
  dh[1][0] = vc * uc;
  dh[1][1] = vc * vc;
  const rd r2 = dh[0][0] + dh[1][1];
  const rd distor = one + two * kd1 * r2;
  const rd distor1_2 = rsqrt_(distor);
  const rd distor3_2 = distor1_2 * distor;
  const rd scale = rd(-2.0) * kd1 / distor3_2;
  for (int i = 0; i < 2; ++i)
    for (int j = 0; j < 2; ++j) dh[i][j] = dh[i][j] * scale;
  dh[0][0] = dh[0][0] + (one / distor1_2);
  dh[1][1] = dh[1][1] + (one / distor1_2);
  for (int i = 0; i < 2; ++i)
    for (int j = 0; j < 3; ++j) {
      rd s(0.0);
      for (int k = 0; k < 2; ++k) s = s + dh[i][k] * du[k][j];
      J[i][j] = s;
    }
}

// The mirror of patch_warp_source for the normal alignment (normals.cu): template pixel (db, da) (column, row offset
// from the centre) of the camera at xo, through the plane through y with normal nW (nd = nW . (y - xo[0:3]), nE1 /
// nE2 = E1 / E2 . (y - xo[0:3])), into the camera at x (RRW = pose_RRW(x)): p_o = ho + (db, da); d_o = adjo
// unproject_point(p_o); den = nW . d_o; t = nd / den; zc = RRW ((xo[0:3] + t d_o) - x[0:3]); g = project(zc) (J =
// dh/dz); Jw = J (RRW d_o); t_a = (nE1 - t (E1 . d_o)) / den, t_b likewise with E2.  True when t is finite and > 0 and
// zc[2] > 0.
struct PatchFwd {
  rd g[2], Jw[2], ta, tb;
};
__device__ __forceinline__ bool patch_warp_forward(const double *cam, const rd adjo[3][3], const rd ho[2],
                                                   const double *xo, const rd RRW[3][3], const double *x,
                                                   const PatchBasis &b, const rd nW[3], rd nd, rd nE1, rd nE2, int db,
                                                   int da, PatchFwd &o) {
  const rd p[2] = {ho[0] + rd((double)db), ho[1] + rd((double)da)};
  rd c[3], dO[3];
  unproject_point(cam, p, c);
  mat3_vec(adjo, c, dO);
  const rd den = dot3(nW, dO);
  const rd t = nd / den;
  rd e[3], zc[3], w[3], J[2][3];
  for (int i = 0; i < 3; ++i) e[i] = (rd(xo[i]) + t * dO[i]) - rd(x[i]);
  mat3_vec(RRW, e, zc);
  project(cam, zc, o.g, J);
  mat3_vec(RRW, dO, w);
  for (int i = 0; i < 2; ++i) o.Jw[i] = (J[i][0] * w[0] + J[i][1] * w[1]) + J[i][2] * w[2];
  o.ta = (nE1 - t * dot3(b.E1, dO)) / den;
  o.tb = (nE2 - t * dot3(b.E2, dO)) / den;
  return isfinite(t.v) && t.v > 0.0 && zc[2].v > 0.0;
}

// Camera::MeasurementNoise, camera.cpp:282-300: R = var I
__device__ __forceinline__ rd measurement_noise(const double *cam, const rd h[2]) {
  const rd u0(cam[4]), v0(cam[5]), sd(cam[7]), one(1.0);
  const rd dx = h[0] - u0, dy = h[1] - v0;
  const rd distance = rsqrt_(dx * dx + dy * dy);
  const rd max_distance = rsqrt_(u0 * u0 + v0 * v0);
  const rd ratio = distance / max_distance;
  const rd sd_use = sd * (one + ratio);
  return one * (sd_use * sd_use);
}

// FeatureModel::func_Si, feature_model.cpp:99-116, for a feature state of NY entries (3: map feature, 6: ray).
// dh_by_dxv = [dh_by_dxp | 0(2x6)] (motion_model.cpp:224-235), so terms with k >= 7 are exact zeros and are
// skipped.  Column-major blocks: Pxx (7 x 7 used) with leading dimension ldxx, Pxy (7 x NY used) ldxy, Pyy ldyy.
template <int NY>
__device__ __forceinline__ void func_Si(const rd dxp[2][7], const rd dy[2][NY], rd var, const double *Pxx,
                                        int ldxx, const double *Pxy, int ldxy, const double *Pyy, int ldyy,
                                        rd S[2][2]) {
  rd A[2][7], Bm[2][NY], Cm[2][NY];
  for (int r = 0; r < 2; ++r) {
    for (int j = 0; j < 7; ++j) {
      rd s(0.0);
      for (int k = 0; k < 7; ++k) s = s + dxp[r][k] * rd(Pxx[k + (size_t)ldxx * j]);
      A[r][j] = s;
    }
    for (int j = 0; j < NY; ++j) {
      rd s(0.0);
      for (int k = 0; k < 7; ++k) s = s + dxp[r][k] * rd(Pxy[k + (size_t)ldxy * j]);
      Bm[r][j] = s;
      rd t(0.0);
      for (int k = 0; k < NY; ++k) t = t + dy[r][k] * rd(Pyy[k + (size_t)ldyy * j]);
      Cm[r][j] = t;
    }
  }
  for (int r = 0; r < 2; ++r)
    for (int c = 0; c < 2; ++c) {
      rd s1(0.0), t1(0.0), t1t(0.0), s4(0.0);
      for (int k = 0; k < 7; ++k) s1 = s1 + A[r][k] * dxp[c][k];
      for (int k = 0; k < NY; ++k) t1 = t1 + Bm[r][k] * dy[c][k];
      for (int k = 0; k < NY; ++k) t1t = t1t + Bm[c][k] * dy[r][k];
      for (int k = 0; k < NY; ++k) s4 = s4 + Cm[r][k] * dy[c][k];
      rd v = rd(0.0) + s1;
      v = v + t1;
      v = v + t1t;
      v = v + s4;
      v = v + (r == c ? var : rd(0.0));
      S[r][c] = v;
    }
}

// The measurement prediction of map feature yi from the camera state xv (monoslam.cpp:289-308): h, dh/dxp, dh/dy,
// R = var I, S; depth = the camera-frame depth of yi (not part of the reference's prediction).
struct FeatPred {
  rd h[2];
  rd dxp[2][7];
  rd dy[2][3];
  rd var;
  rd S[2][2];
  rd depth;
};

// The measurement model of map feature yi seen from the camera pose xp (7: r, q): h, dh/dxp, dh/dy and the
// camera-frame depth of yi (monoslam.cpp:289-308 without R and S).  predict_feature and iterate_kernel (iterate.cu)
// both evaluate the model here.
__device__ __forceinline__ void measure_feature(const double *cam, const double *xp, const rd yi[3], rd h[2],
                                                rd dxp[2][7], rd dy[2][3], rd &depth) {
  rd z[3], dz_dxp[3][7], RRW[3][3], J[2][3];
  zeroedyi(yi, xp, z, dz_dxp, RRW);
  project(cam, z, h, J);
  for (int i = 0; i < 2; ++i) {
    for (int j = 0; j < 7; ++j) {
      rd s(0.0);
      for (int k = 0; k < 3; ++k) s = s + J[i][k] * dz_dxp[k][j];
      dxp[i][j] = s;
    }
    for (int j = 0; j < 3; ++j) {
      rd s(0.0);
      for (int k = 0; k < 3; ++k) s = s + J[i][k] * RRW[k][j];
      dy[i][j] = s;
    }
  }
  depth = z[2];
}

// Pxx: shared 13x13 col-major; Pcol: global pointer to P(0, pos) (column-major, ld)
__device__ void predict_feature(const double *cam, const double *xv, const rd yi[3],
                                const double *Pxx, const double *Pcol, int ld, int pos,
                                FeatPred &o) {
  measure_feature(cam, xv, yi, o.h, o.dxp, o.dy, o.depth);
  o.var = measurement_noise(cam, o.h);
  func_Si<3>(o.dxp, o.dy, o.var, Pxx, 13, Pcol, ld, Pcol + pos, ld, o.S);
}

// (S^-1)00, 01, 11 of a 2x2 S: LLT, L^-1 in closed form, L^-T L^-1 (monoslam.cpp:371-374; Particle::set_S,
// feature_init_info.cpp:57-65; the oracle's puinv_from_S)
__device__ __forceinline__ void sinv_from_S(rd s00, rd s10, rd s11, rd Sinv[3]) {
  const rd l00 = rsqrt_(s00);
  const rd l10 = s10 / l00;
  const rd l11 = rsqrt_(s11 - l10 * l10);
  const rd x00 = rd(1.0) / l00;
  const rd x10 = (rd(0.0) - l10 * x00) / l11;
  const rd x11 = rd(1.0) / l11;
  Sinv[0] = x00 * x00 + x10 * x10;
  Sinv[1] = x10 * x11;
  Sinv[2] = x11 * x11;
}

// stream s's camera row into the block's shared copy sc (one double per thread); read it after a __syncthreads()
__device__ __forceinline__ void load_stream_cam(const Sl2Dev &d, int s, Sl2StreamCam &sc) {
  const int tid = threadIdx.x;
  if (tid < (int)(sizeof(Sl2StreamCam) / sizeof(double)))
    reinterpret_cast<double *>(&sc)[tid] = reinterpret_cast<const double *>(d.cams + s)[tid];
}

// the reprojection inlier test of a match: the map point y seen from the pose xp (RRW = pose_RRW(xp)) lies in front
// of the camera and d2 = |z - h(y)|^2 <= t2 (NaN: never); *d2 is written only for a point in front
__device__ __forceinline__ bool reproj_inlier(const double *cam, const rd RRW[3][3], const double *xp, const rd y[3],
                                              const double z[2], double t2, double *d2) {
  rd dd[3], zc[3], g[2], uc, vc;
  zeroed_point(RRW, y, xp, dd, zc);
  if (!(zc[2].v > 0.0)) return false;
  project_point(cam, zc, g, uc, vc);
  const rd du = rd(z[0]) - g[0], dv = rd(z[1]) - g[1];
  *d2 = (du * du + dv * dv).v;
  return *d2 <= t2;
}

// The support of one hypothesis, one warp: lane takes the matches j = lane + 32 c of the k, in_fn(j) decides each.
// Returns how many are in; lane 0 writes the inlier words mask[c], unless mask is the literal nullptr (count only).
template <typename Mask, typename InFn>
__device__ __forceinline__ int warp_support(int k, int lane, Mask mask, InFn in_fn) {
  int sup = 0;
  for (int c32 = 0; c32 * 32 < k; ++c32) {
    const int j = c32 * 32 + lane;
    const unsigned b = __ballot_sync(0xffffffffu, j < k && in_fn(j));
    if constexpr (!std::is_null_pointer<Mask>::value)
      if (lane == 0) mask[c32] = b;
    sup += __popc(b);
  }
  return sup;
}

}  // namespace
