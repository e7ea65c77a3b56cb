// update.cu — EKF update on sm_90a as a pipeline of five kernels (all streams of a context per launch).
//
// Replaces, per camera stream:
//   Kalman::KalmanFilterUpdate             kalman.cpp:72-119  (+ gather/scatter monoslam.cpp:501-614)
//   MonoSLAM::normalise_state + symmetrise monoslam.cpp:616-637, 143-150
//   attempt / success bookkeeping          monoslam.cpp:479-496
//
// Mathematically the reference's  K = P H^T S^-1,  x += K nu,  P -= K S K^T  with S = H P H^T + R:
//   S = U^T U (Cholesky),  Y = U^-T (H P),  w = U^-T nu   =>   x += Y^T w,   P -= Y^T Y.
// H is structurally sparse (7 + 3 non-zero columns per row) and is never formed.
//
//   kernel           grid                      work per CTA
//   upd_hp / upd_hp2 streams                   measurement list; G = [ S | H P | nu ] (m x (m+n+1), row-major scratch):
//                                              a stream over P, thread = state column, 16 (upd_hp2: 8, double-buffered)
//                                              rows of H P per block, S = (H P) H^T + R from the block's rows in shared
//                                              memory (upd_hp2: under the loads of the next block).
//   upd_chol         streams                   blocked Cholesky of the S part only (16-row panels, left-looking with
//                                              a look-ahead for the next diagonal block) -> U in place, and
//                                              W_pp = U_pp^-T of every panel.  The serial chain of the update
//                                              lives here and touches 200 x 200 numbers, not 200 x 514.
//   upd_solve        streams (x column slabs)  Y = U^-T [H P | nu]: a warp pair owns 8 columns and keeps all m rows
//                                              of them in REGISTERS (DMMA fragment layout); U and the W_pp arrive
//                                              by bulk copies on mbarriers, once per CTA; the product runs on the
//                                              FP64 tensor path, every tile of Y formed once, no per-tile guards
//                                              when the rows reach the last panel.  Column groups are independent.
//   upd_syrk         64x64 tiles x streams     P -= Y^T Y (upper tiles computed, lower mirrored; a diagonal tile
//                                              computes its 8x8 blocks on / above the diagonal); the nu column rides
//                                              along as column n of Y, so the tile row that holds it yields
//                                              x += Y^T w in its epilogue.
//   upd_finish       streams                   normalise_state, symmetrise, counters.
//
// Every kernel starts with pdl_prologue(): launched with the PDL attribute (sl2_use_pdl: a single camera stream) the
// eight kernels of a step overlap their launch latencies; without it the two instructions do nothing.
//
// Every re-read of the round-1 single-kernel design (finished rows of G gathered from L2/HBM by every panel over
// all 514 columns, Y slabs re-staged per tile by a CTA that owns the whole stream) is gone: G is written once and
// read once by upd_solve (registers), Y is written once and read by the tiles of the same stream, which run at the
// same time on neighbouring SMs (L2 hits).  The dense O(n^2 m) parts use ordinary FP64 FMAs / DMMA (tolerance
// 1e-5 relative, north star); nothing in this file decides which pixels are searched.
#include <type_traits>

#include "sl2_common.cuh"
#include "sl2_ptx.cuh"

namespace {

constexpr int UPD_THREADS = 256;
constexpr int UPD_NB = 16;   // Cholesky row-panel height (two DMMA M-tiles)
constexpr int UPD_WS = 20;   // row stride of the W table
constexpr int UPD_DS = 20;   // row stride of the diagonal-block scratch (conflict-free fragments)
constexpr int UPD_MS = 20;   // row stride of the multiplier table: 32 B (mod 128) => conflict-free A fragments
constexpr int UPD_YS = 68;   // padded row stride of a staged Y slab (doubles): conflict-free DMMA reads
constexpr int SOLVE_MAX_WARPS = 8;   // warps (8-column groups) per upd_solve CTA: 2 per SM sub-partition, <= 255 registers

// Every measurement-sized table below is sized from kmax = Sl2Dev::kmax (features one step can measure), never from
// the map capacity: S and its factor live in shared memory, H P rows and P in HBM.
__host__ __device__ inline int upd_keven(int kmax) { return (kmax + 1) & ~1; }
__host__ __device__ inline int upd_panw(int kmax) {
  // panel buffer of the factor kernel: S columns only; row stride = 2 (mod 16) doubles: the 8 rows of a DMMA
  // C fragment hit distinct banks
  return ((2 * upd_keven(kmax) + 15) & ~15) + 2;
}
__host__ __device__ inline size_t upd_pan_doubles(int kmax) { return (size_t)UPD_NB * upd_panw(kmax); }

// D(8x8) = A(8x4) * B(4x8) + C on the FP64 tensor path: lane holds A(lane/4, lane%4),
// B(lane%4, lane/4) and C(lane/4, 2*(lane%4) + {0,1}).
__device__ __forceinline__ void dmma884(double &c0, double &c1, double a, double b) {
  asm("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
      : "+d"(c0), "+d"(c1)
      : "d"(a), "d"(b));
}
// D(16x8) = A(16x4) * B(4x8) + C: lane (g, t) = (lane/4, lane%4) holds A(g + 8 i, t) in a[i], B(t, g) in b and
// C(g + 8 (e/2), 2 t + e%2) in c[e].
__device__ __forceinline__ void dmma1684(double (&c)[4], const double (&a)[2], double b) {
  asm("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
      : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
      : "d"(a[0]), "d"(a[1]), "d"(b));
}
// D(16x8) = A(16x8) * B(8x8) + C: lane (g, t) = (lane/4, lane%4) holds A(g + 8 (i%2), t + 4 (i/2)) in a[i],
// B(t + 4 i, g) in b[i] and C(g + 8 (e/2), 2 t + e%2) in c[e].
__device__ __forceinline__ void dmma1688(double (&c)[4], const double (&a)[4], const double (&b)[2]) {
  asm("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
      : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
// bulk copy (cp.async.bulk): the TMA engine moves a contiguous run of bytes global -> shared and reports completion
// as transaction bytes on an mbarrier; one instruction per row, no per-chunk index math.
// bytes: multiple of 16; dst / src 16-byte aligned
__device__ __forceinline__ void bulk_g2s(void *smem_dst, const void *gsrc, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(bar)
               : "memory");
}

// 1/sqrt(d) for a positive pivot: MUFU seed + two Newton steps (about 1 ulp); a handful of FP64
// instructions instead of the library routine -- this sits on the serial path of every panel.
__device__ __forceinline__ double pivot_rsqrt(double dv) {
  double y;
  asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(dv));
#pragma unroll
  for (int it = 0; it < 2; ++it) {
    const double e = fma(-(dv * y), y, 1.0);
    y = fma(0.5 * y, e, y);
  }
  return y;
}

// One warp: Cholesky of the 8x8 block at (o, o) of dg (upper triangle, U^T U = A) and W = U^-T into
// the same block of Wm.  Lane j (mod 8) holds column j of A and column j of W in registers.  Per pivot r:
// the pivot travels by one shuffle, 1/u_rr is computed by every lane (uniform), row r of U is a[r] / u_rr,
// and each multiplier U(r, i) (one more shuffle) updates a[i] AND w[i]: W is the forward elimination of the
// identity with the same multipliers (row_i -= U(r,i) * row_r), so it costs no shuffles and no serial tail.
// All 32 lanes must call.  (Measured alternative, same bits: every lane factoring its own copy of the whole block
// row by row with no shuffle at all -- 156 FP64 instructions per block instead of 136 + 36 shuffles -- left the
// batched kernel unchanged and made the single-stream factor slower; so did dropping the second Newton step of the
// pivot's rsqrt: with a full batch the panel's trailing update, fed from L2, is what the barrier waits for, not the
// factor.)
__device__ __forceinline__ void chol8_inv(double *dg, double *Wm, int o, int lane) {
  const int j = lane & 7;
  double a[8], w[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    a[i] = (i <= j) ? dg[(o + i) * UPD_DS + o + j] : 0.0;
    w[i] = (i == j) ? 1.0 : 0.0;
  }
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    const double dv = __shfl_sync(0xffffffffu, a[r], r);
    const double iu = pivot_rsqrt(dv);
    const double urj = a[r] * iu;  // lane r: d / sqrt(d) = u_rr
    a[r] = urj;
    w[r] *= iu;
#pragma unroll
    for (int i = r + 1; i < 8; ++i) {
      const double uri = __shfl_sync(0xffffffffu, urj, i);
      a[i] -= uri * urj;
      w[i] -= uri * w[r];
    }
  }
  __syncwarp();  // every lane has read its (mirrored) column before the block is overwritten
  if (lane < 8) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (i <= j) dg[(o + i) * UPD_DS + o + j] = a[i];
      Wm[(o + i) * UPD_WS + o + j] = w[i];
    }
  }
}

// =============================================================================================
// kernel 0: upd_hp / upd_hp2 — measurement list, G = [ S | H P | nu ]: streams P once, one thread per state column
// =============================================================================================
// H has 7 (fused step: dh/dxv = [dh/dxp | 0]) or 13 (staged API) dense columns and 3 structural dh/dy columns per
// row, so   (H P)(i, j) = sum_k Hx(i, k) P(k, j) + sum_c Hy(i, c) P(pos_i + c, j):
// for the two rows of one measured feature that is three rows of P (contiguous along j, P symmetric) read exactly
// once, plus the 13 leading rows of P, which a thread keeps in registers for its column j.  The kernel is a stream
// over P (0.75 MB in, 0.5 MB H P + S out per 100-feature stream) with ~16 FMAs per element, so it is laid out for
// the memory system: thread = column (8 B x 32 lanes = whole lines), all 24 row loads of an 8-feature block in
// flight before the first FMA, H rows broadcast from shared memory.  (The round-2 first version ran the 13 dense
// columns on DMMA tiles and gathered P into fragments: L1 request bound.  Measured on this version:
// prefetch.global.L2 of the next block's rows before the S phase made it slower.)
// The CTA's 16 rows of H P also stay in shared memory for S = (H P) H^T + R: thread = measurement column i',
// H(i', :) in registers, dense part from broadcast reads, structural part gathered from the rows.
constexpr int HP_THREADS = 320;
constexpr int HP_ROWS = 16;   // measurement rows per block of upd_hp (8 features); upd_hp2: two buffers of 8 rows
constexpr int HP_HRS = 18;    // row stride of the H table: [13 dense | 3 dh/dy | 2 pad] doubles (16 B aligned rows)
struct HpSmem {
  double *Hrow;  // [mmax][HP_HRS]
  double *Rv;    // [K][3]  (R00, R01, R11)
  double *nu;    // [mmax]
  double *hprow; // [HP_ROWS][ld]  H P rows of the running block (upd_hp2: of the two blocks in flight)
  int *mfeat;    // [K]
  int *wcount;   // [16]
  double *park;  // [KD][HP_THREADS]  upd_hp2 only: the KD leading rows of P, one column per thread
};
// The one layout of that shared memory, for the launcher (bytes) and the kernels (hp_carve): byte offsets of the
// tables in the order above.  K = upd_keven(kmax) is even, so hprow is 16-byte aligned and park 8-byte aligned.
// kd_park = KD for upd_hp2, 0 for upd_hp.
struct HpLayout {
  size_t Hrow, Rv, nu, hprow, mfeat, wcount, park, bytes;
};
__host__ __device__ inline HpLayout hp_layout(int kmax, int ld, int kd_park) {
  const size_t K = upd_keven(kmax);
  HpLayout l;
  l.Hrow = 0;
  l.Rv = l.Hrow + 2 * K * HP_HRS * sizeof(double);
  l.nu = l.Rv + 3 * K * sizeof(double);
  l.hprow = l.nu + 2 * K * sizeof(double);
  l.mfeat = l.hprow + (size_t)HP_ROWS * ld * sizeof(double);
  l.wcount = l.mfeat + K * sizeof(int);
  l.park = l.wcount + 16 * sizeof(int);
  l.bytes = l.park + (size_t)kd_park * HP_THREADS * sizeof(double);
  return l;
}
__device__ __forceinline__ HpSmem hp_carve(uint8_t *base, int kmax, int ld) {
  const HpLayout l = hp_layout(kmax, ld, 0);
  HpSmem u;
  u.Hrow = reinterpret_cast<double *>(base + l.Hrow);
  u.Rv = reinterpret_cast<double *>(base + l.Rv);
  u.nu = reinterpret_cast<double *>(base + l.nu);
  u.hprow = reinterpret_cast<double *>(base + l.hprow);
  u.mfeat = reinterpret_cast<int *>(base + l.mfeat);
  u.wcount = reinterpret_cast<int *>(base + l.wcount);
  u.park = reinterpret_cast<double *>(base + l.park);
  return u;
}

// Measurement list in selected order (successful only, monoslam.cpp:556-571) and the H rows, R, nu of every
// measurement into shared memory; returns K (measured features) or -1 when this CTA has no row block (rows_per_block
// rows per block, block index blockIdx.x).  Every CTA of the stream pays this prologue.  All threads must call.
__device__ __forceinline__ int hp_tables(const Sl2Dev &d, const HpSmem &sm, int s, int rows_per_block, int staged_m,
                                         const int *st_feat, const double *st_Hxv, const double *st_Hy,
                                         const double *st_R, const double *st_nu) {
  const int tid = threadIdx.x;
  const size_t fb = (size_t)s * d.Nmax;
  // ---- measurement list in selected order, successful only (monoslam.cpp:556-571) --------------
  int K;
  if (staged_m >= 0) {
    K = staged_m / 2;
    for (int k = tid; k < K; k += HP_THREADS) sm.mfeat[k] = st_feat[k];
  } else {
    const int nsel = d.nsel[s];
    int feat = -1;
    if (tid < d.Nmax && tid < nsel) {
      const int i = d.job_feat[fb + tid];
      if (i >= 0 && d.found[fb + i] == 1) feat = i;
    }
    // nsel <= kmax: the warps beyond the first (SL2_MAX_MEASURED + 31) / 32 select nothing
    K = block_gather(feat, sm.mfeat, sm.wcount, (SL2_MAX_MEASURED + 31) / 32);
  }
  const int m = 2 * K;
  if (blockIdx.x == 0 && tid == 0) {
    d.upd_m[s] = m;
    if (staged_m < 0) d.nmeas[s] = K;
  }
  if (rows_per_block * (int)blockIdx.x >= m) return -1;
  for (int e = tid; e < m * HP_HRS; e += HP_THREADS) sm.Hrow[e] = 0.0;
  __syncthreads();
  // ---- H rows, R, nu of every measurement (every CTA of the stream pays this prologue) -------------------
  if (staged_m >= 0) {
    for (int e = tid; e < m * 13; e += HP_THREADS) {
      const int i = e / 13, c = e - i * 13;
      sm.Hrow[i * HP_HRS + c] = st_Hxv[e];
    }
    for (int e = tid; e < K * 6; e += HP_THREADS) {
      const int i = e / 3, c = e - i * 3;
      sm.Hrow[i * HP_HRS + 13 + c] = st_Hy[e];
    }
    for (int e = tid; e < m; e += HP_THREADS) sm.nu[e] = st_nu[e];
    for (int k = tid; k < K; k += HP_THREADS) {
      // R_k 2x2 column-major (symmetric; the host entry point rejects R01 != R10)
      sm.Rv[k * 3 + 0] = st_R[k * 4 + 0];
      sm.Rv[k * 3 + 1] = st_R[k * 4 + 2];
      sm.Rv[k * 3 + 2] = st_R[k * 4 + 3];
    }
  } else {
    for (int e = tid; e < K * 14; e += HP_THREADS) {  // dh/dxv = [dh/dxp | 0] (motion_model.cpp:224-235)
      const int k = e / 14, q = e - k * 14, r = q >= 7;
      sm.Hrow[(2 * k + r) * HP_HRS + q - 7 * r] = d.dh_dxp[(fb + sm.mfeat[k]) * 14 + q];
    }
    for (int e = tid; e < K * 6; e += HP_THREADS) {
      const int i = e / 3, c = e - i * 3;
      sm.Hrow[i * HP_HRS + 13 + c] = d.dh_dy[(fb + sm.mfeat[i >> 1]) * 6 + (i & 1) * 3 + c];
    }
    for (int e = tid; e < m; e += HP_THREADS) {
      const size_t f = fb + sm.mfeat[e >> 1];
      // nu = z - h (full_feature_model.cpp:197-200), z = (double)(u,v) (monoslam.cpp:382-383)
      sm.nu[e] = (rd((double)d.z_uv[f * 2 + (e & 1)]) - rd(d.h[f * 2 + (e & 1)])).v;
    }
    for (int k = tid; k < K; k += HP_THREADS) {
      const double var = d.Rvar[fb + sm.mfeat[k]];  // R_i = var * I (camera.cpp:294-299)
      sm.Rv[k * 3 + 0] = var;
      sm.Rv[k * 3 + 1] = 0.0;
      sm.Rv[k * 3 + 2] = var;
    }
  }
  __syncthreads();

  return K;
}

// ---- the per-block steps of upd_hp and upd_hp2: the two kernels differ only in the loop around them -------------
// The KD leading rows of P for state column j (zero past the last column n).
template <int KD>
__device__ __forceinline__ void hp_load_dense(double (&Pd)[KD], const double *__restrict__ P, int ld, int j, int n) {
#pragma unroll
  for (int k = 0; k < KD; ++k) Pd[k] = j < n ? P[(size_t)k * ld + j] : 0.0;
}

// The 3 structural rows of P of the F features from k0 on, column j: every load of the block in flight at once.
template <int F>
__device__ __forceinline__ void hp_load_struct(double (&pv)[F][3], const HpSmem &sm, const double *__restrict__ P,
                                               int ld, int j, int n, int k0, int K) {
#pragma unroll
  for (int f = 0; f < F; ++f) {
    const int kk = k0 + f;
    const int pos = SL2_NXV + 3 * sm.mfeat[kk < K ? kk : 0];
#pragma unroll
    for (int c = 0; c < 3; ++c) pv[f][c] = (kk < K && j < n) ? P[(size_t)(pos + c) * ld + j] : 0.0;
  }
}

// (H P)(i, j) of one measurement row (hrow = its H row in shared memory): the KD dense terms in pairs of H entries,
// then the 3 structural terms.
template <int KD>
__device__ __forceinline__ double hp_row_value(const double *hrow, const double (&Pd)[KD], const double (&pv)[3]) {
  const double2 *hr = reinterpret_cast<const double2 *>(hrow);
  double acc = 0.0;
#pragma unroll
  for (int k2 = 0; k2 < (KD + 1) / 2; ++k2) {
    const double2 hv = hr[k2];
    acc += hv.x * Pd[2 * k2];
    if (2 * k2 + 1 < KD) acc += hv.y * Pd[2 * k2 + 1];
  }
  const double2 hy0 = hr[6], hy1 = hr[7];  // columns 12..15: (dense 12 | dh/dy 0..2)
  acc += hy0.y * pv[0];
  acc += hy1.x * pv[1];
  acc += hy1.y * pv[2];
  return acc;
}

// H P of the 2 F rows of the block from row0 on, column j: to G and to the block's rows in shared memory (buf,
// row stride ld).
template <int F, int KD>
__device__ __forceinline__ void hp_block_rows(const HpSmem &sm, const double (&Pd)[KD], const double (&pv)[F][3],
                                              double *__restrict__ G, int ldg, double *__restrict__ buf, int ld,
                                              int row0, int K, int j, int n) {
  const int m = 2 * K, k0 = row0 >> 1;
#pragma unroll
  for (int f = 0; f < F; ++f) {
    if (k0 + f < K) {  // CTA-uniform
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int i = row0 + 2 * f + r;
        const double acc = hp_row_value(sm.Hrow + (size_t)i * HP_HRS, Pd, pv[f]);
        if (j < n) {
          G[(size_t)i * ldg + m + j] = acc;
          buf[(size_t)(2 * f + r) * ld + j] = acc;
        }
      }
    }
  }
}

// The nu column of the block's rows: G(i, m + n) = nu_i.
__device__ __forceinline__ void hp_store_nu(const HpSmem &sm, double *__restrict__ G, int ldg, int m, int n, int row0,
                                            int rows) {
  const int tid = threadIdx.x;
  if (tid < rows) G[(size_t)(row0 + tid) * ldg + m + n] = sm.nu[row0 + tid];
}

// S = (H P) H^T + R for the rows row0 .. row0 + rows - 1 (rows <= R) of a block, columns from the row's own feature
// on: thread = measurement column i', H(i', :) in registers, the block's H P rows from shared memory (buf, row stride
// ld; dense columns read as 16-byte pairs), four rows at a time (independent accumulation chains: a single chain is
// 10-16 dependent FMAs per entry).
template <int R, int KD>
__device__ __forceinline__ void hp_s_rows(const HpSmem &sm, const double *__restrict__ buf, int ld,
                                          double *__restrict__ G, int ldg, int m, int row0, int rows) {
  for (int ip = threadIdx.x; ip < m; ip += HP_THREADS) {
    if (ip < row0) continue;
    const int kp = ip >> 1, rp = ip & 1;
    const double2 *hr = reinterpret_cast<const double2 *>(sm.Hrow + (size_t)ip * HP_HRS);
    double hd[KD + 1];
#pragma unroll
    for (int k2 = 0; k2 < (KD + 1) / 2; ++k2) {
      const double2 hv = hr[k2];
      hd[2 * k2] = hv.x;
      hd[2 * k2 + 1] = hv.y;
    }
    const double2 hy0 = hr[6], hy1 = hr[7];
    const double hys[3] = {hy0.y, hy1.x, hy1.y};
    const int pos = SL2_NXV + 3 * sm.mfeat[kp];
    const double r_same = sm.Rv[kp * 3 + 2 * rp], r_cross = sm.Rv[kp * 3 + 1];
#pragma unroll
    for (int il0 = 0; il0 < R; il0 += 4) {
      if (il0 < rows) {
        double acc[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[q] = 0.0;
#pragma unroll
        for (int c2 = 0; c2 < KD / 2; ++c2)
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const double2 v = *reinterpret_cast<const double2 *>(buf + (size_t)(il0 + q) * ld + 2 * c2);
            acc[q] += v.x * hd[2 * c2];
            acc[q] += v.y * hd[2 * c2 + 1];
          }
        if (KD & 1) {
#pragma unroll
          for (int q = 0; q < 4; ++q) acc[q] += buf[(size_t)(il0 + q) * ld + KD - 1] * hd[KD - 1];
        }
#pragma unroll
        for (int c = 0; c < 3; ++c)
#pragma unroll
          for (int q = 0; q < 4; ++q) acc[q] += buf[(size_t)(il0 + q) * ld + pos + c] * hys[c];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int i = row0 + il0 + q;
          if (il0 + q < rows && ip >= (i & ~1)) {
            if ((i >> 1) == kp) acc[q] += (i == ip) ? r_same : r_cross;
            G[(size_t)i * ldg + ip] = acc[q];
          }
        }
      }
    }
  }
}

// KD = dense columns of H that can be nonzero (7: fused step, 13: staged)
template <int KD>
__global__ void __launch_bounds__(HP_THREADS, 2) upd_hp_kernel(
    const Sl2Dev d, int stream_lo, int staged_m, const int *st_feat, const double *st_Hxv,
    const double *st_Hy, const double *st_R, const double *st_nu) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  pdl_prologue();
  const int ld = d.ld, ldg = d.ldg;
  const HpSmem sm = hp_carve(smem_raw, d.kmax, ld);
  const int s = stream_lo + blockIdx.y;
  const int tid = threadIdx.x;
  const int n = SL2_NXV + 3 * d.nfeat[s];
  const double *__restrict__ P = d.P + (size_t)s * ld * ld;
  double *__restrict__ G = d.G + (size_t)s * d.mmax * ldg;
  const int K = hp_tables(d, sm, s, HP_ROWS, staged_m, st_feat, st_Hxv, st_Hy, st_R, st_nu);
  if (K < 0) return;
  const int m = 2 * K;

  constexpr int FB = HP_ROWS / 2;            // features per block
  const int nch = (n + HP_THREADS - 1) / HP_THREADS;  // column chunks (1 up to 102 features)
  double Pd[KD];
  if (nch == 1) hp_load_dense(Pd, P, ld, tid, n);
  // row blocks blockIdx.x, blockIdx.x + gridDim.x, ...: the measurement list and the H tables are built once
  for (int rb = blockIdx.x; HP_ROWS * rb < m; rb += gridDim.x) {
    const int row0 = HP_ROWS * rb, rows = min(HP_ROWS, m - row0);
    for (int ch = 0; ch < nch; ++ch) {
      const int j = ch * HP_THREADS + tid;
      if (nch > 1) hp_load_dense(Pd, P, ld, j, n);
      double pv[FB][3];
      hp_load_struct(pv, sm, P, ld, j, n, row0 >> 1, K);
      hp_block_rows(sm, Pd, pv, G, ldg, sm.hprow, ld, row0, K, j, n);
    }
    hp_store_nu(sm, G, ldg, m, n, row0, rows);
    __syncthreads();
    hp_s_rows<HP_ROWS, KD>(sm, sm.hprow, ld, G, ldg, m, row0, rows);
    __syncthreads();  // hprow of this block is rewritten by the next one
  }
}

// upd_hp, software-pipelined (maps of up to (HP_THREADS - 13) / 3 features): the same stream over P in 8-row blocks
// (4 features) with the shared-memory rows of H P double-buffered, so that
//   loads of block b+1 issued  ->  S = (H P) H^T + R of block b from shared memory  ->  FMAs / stores of block b+1
// and the structural row loads (the HBM stream) are in flight WHILE the S phase runs instead of after it; one
// __syncthreads per block.  The per-block steps are upd_hp's, so the results are identical.
template <int KD>
__global__ void __launch_bounds__(HP_THREADS, 2) upd_hp2_kernel(
    const Sl2Dev d, int stream_lo, int staged_m, const int *st_feat, const double *st_Hxv,
    const double *st_Hy, const double *st_R, const double *st_nu) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  pdl_prologue();
  constexpr int R2 = HP_ROWS / 2, F2 = R2 / 2;  // rows / features per block
  const int ld = d.ld, ldg = d.ldg;
  const HpSmem sm = hp_carve(smem_raw, d.kmax, ld);
  const int s = stream_lo + blockIdx.y;
  const int tid = threadIdx.x;
  const int n = SL2_NXV + 3 * d.nfeat[s];
  const double *__restrict__ P = d.P + (size_t)s * ld * ld;
  double *__restrict__ G = d.G + (size_t)s * d.mmax * ldg;
  const int K = hp_tables(d, sm, s, R2, staged_m, st_feat, st_Hxv, st_Hy, st_R, st_nu);
  if (K < 0) return;
  const int m = 2 * K;
  const int j = tid;  // this thread's state column (n <= HP_THREADS: the launcher's condition)
  // the KD leading rows of P for this thread's column: parked in shared memory (own slot per thread, no barrier
  // needed) so that they do not occupy registers during the S phase, when the 12 structural loads are in flight
  double *const park = sm.park + tid;
  {
    double Pd[KD];
    hp_load_dense(Pd, P, ld, j, n);
#pragma unroll
    for (int k = 0; k < KD; ++k) park[k * HP_THREADS] = Pd[k];
  }
  double pv[F2][3];
  auto consume = [&](int rb, double *__restrict__ buf) {  // H P of block rb -> G and the shared rows
    const int row0 = R2 * rb;
    double Pd[KD];
#pragma unroll
    for (int k = 0; k < KD; ++k) Pd[k] = park[k * HP_THREADS];
    hp_block_rows(sm, Pd, pv, G, ldg, buf, ld, row0, K, j, n);
    hp_store_nu(sm, G, ldg, m, n, row0, min(R2, m - row0));
  };
  auto sphase = [&](int rb, const double *__restrict__ buf) {
    hp_s_rows<R2, KD>(sm, buf, ld, G, ldg, m, R2 * rb, min(R2, m - R2 * rb));
  };
  int rb = blockIdx.x, par = 0;
  double *const buf0 = sm.hprow, *const buf1 = sm.hprow + (size_t)R2 * ld;
  hp_load_struct(pv, sm, P, ld, j, n, F2 * rb, K);
  consume(rb, buf0);
  __syncthreads();
  for (;;) {
    const int nb = rb + gridDim.x;
    const bool more = R2 * nb < m;  // CTA-uniform
    if (more) hp_load_struct(pv, sm, P, ld, j, n, F2 * nb, K);
    sphase(rb, par ? buf1 : buf0);
    if (!more) break;
    consume(nb, par ? buf0 : buf1);
    __syncthreads();  // block nb's rows are complete, and nobody still reads the buffer block nb + 1 will take
    rb = nb;
    par ^= 1;
  }
}

// =============================================================================================
// kernel 1: upd_chol — Cholesky of S, finished rows of U in G (L2), two streams per SM
// =============================================================================================
// This kernel is a serial chain: 13 diagonal blocks per stream (m = 200), each factored by ONE warp (~7 k cycles:
// two 8x8 register/shuffle factorizations joined by 8x8 DMMA products), and nothing in the update can start
// before it ends.  What hides it is other streams on the same SM, so it is kept small enough for two CTAs per SM
// (all streams of the benchmark resident at once).  Measured alternative: S / U resident in shared memory
// (193 KB, one CTA per SM, two waves) made every panel faster and the kernel slower.
//
// Left-looking by 16-row panels with a look-ahead, so that the only things between two block factorizations are
// four DMMA k-steps from shared memory and the W * C product of the finished panel:
//   pool of work items per panel p, handed out dynamically to the 8 warps:
//     item 0  (warp 0)  diagonal block of p = pre-updated block (dpre, from the look-ahead of panel p-1) minus the
//                       contribution of panel p-1's 16 rows (multipliers already in shared memory), then factor it
//     item 1            look-ahead for panel p+1: its diagonal block minus the contributions of all rows < i0
//                       (final), into dpre_next; the multipliers it reads on the way go to mult_next
//     items 2..         trailing columns of panel p in batches of 4 / 2 / 1 8-column groups (B fragments from L2,
//                       software pipelined 4 / 8 / 16 k-steps deep: the fewer groups are left, the narrower and deeper)
//   finish (all warps)  U_panel = W * C_panel -> G; the 16 columns that are panel p+1's multipliers -> mult_next
constexpr int CH_D = 4;    // k-steps in flight of the look-ahead item (2 loads per step)
static_assert(4 % CH_D == 0, "nk is a multiple of 4: the look-ahead's pipelined loop runs every k-step");
constexpr int CH_DPS = 18; // row stride of the pre-updated diagonal block

// One batch item of the panel update: GB 8-column groups from group g0 on, C(16 x 8 GB) = S entries - A * B over the
// nk finished k-steps (nk is a multiple of 4); A(r,k) = U(k,i0+r) (negated multipliers, shared memory), B = finished
// rows of U (global / L2), D (4 or 8) k-steps of B fragments in flight.  The result goes to the panel buffer.
// The k loop is kept to a pointer bump, GB loads, 2 shared loads and GB m16n8k4 DMMAs (both 8-row halves of the
// panel in one product) per step: columns past the width are
// loaded like any other (they are columns of H P in the same row: valid memory, finite, and they only reach entries
// of C that are never used), so there is no per-element predicate or index arithmetic in it.
template <int GB, int D>
__device__ __forceinline__ void chol_batch(const double *__restrict__ G, int ldg, const double *__restrict__ mcur,
                                           double *__restrict__ pan, int PW, int i0, int nbp, int nk, int ngroups,
                                           int width, int g0, int lr, int lc) {
  static_assert(D == 4 || D == 8, "nk is a multiple of 4");
  double c[GB][4];  // m16n8 C fragments: c[q][2 mt + e] = C(8 mt + lr, 8 (g0 + q) + 2 lc + e)
#pragma unroll
  for (int q = 0; q < GB; ++q) {
    const int cc = i0 + (g0 + q) * 8 + 2 * lc;  // C fragment: rows lr / lr+8, columns cc, cc+1
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
      const int r = mt * 8 + lr;
      const bool rv = r < nbp && (g0 + q) < ngroups;
      c[q][2 * mt] = (rv && cc < width) ? G[(size_t)(i0 + r) * ldg + cc] : 0.0;
      c[q][2 * mt + 1] = (rv && cc + 1 < width) ? G[(size_t)(i0 + r) * ldg + cc + 1] : 0.0;
    }
  }
  // B fragment of k-step st, group q: G[(4 st + lc) * ldg + i0 + 8 (g0 + q) + lr]
  const size_t kstride = (size_t)4 * ldg;
  const double *gpre = G + (size_t)lc * ldg + i0 + g0 * 8 + lr;  // next k-step to request
  const double *ap = mcur + lc * UPD_MS + lr;                    // A fragments of the next k-step to use
  double b[D][GB];
  auto loadb = [&](double *dst) {
#pragma unroll
    for (int q = 0; q < GB; ++q) dst[q] = gpre[8 * q];
    gpre += kstride;
  };
  auto step = [&](const double *bu) {
    const double a[2] = {ap[0], ap[8]};  // rows lr and 8 + lr of the panel: one m16n8k4 A fragment
    ap += 4 * UPD_MS;
#pragma unroll
    for (int q = 0; q < GB; ++q) dmma1684(c[q], a, bu[q]);
  };
#pragma unroll
  for (int u = 0; u < D - 1; ++u)
    if (u < nk) loadb(b[u]);
  int kb = 0;
  for (; kb + D <= nk; kb += D) {
#pragma unroll
    for (int u = 0; u < D; ++u) {
      if (kb + u + D - 1 < nk) loadb(b[(u + D - 1) % D]);  // warp-uniform
      step(b[u]);
    }
  }
  if (D == 8 && kb < nk) {  // four steps left, their fragments are in flight or landed
#pragma unroll
    for (int u = 0; u < 4; ++u) step(b[u]);
  }
#pragma unroll
  for (int q = 0; q < GB; ++q) {
    if (g0 + q < ngroups) {
      const int pc = (g0 + q) * 8 + 2 * lc;
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
        *reinterpret_cast<double2 *>(pan + (size_t)(mt * 8 + lr) * PW + pc) = make_double2(c[q][2 * mt], c[q][2 * mt + 1]);
    }
  }
}

struct CholSmem {
  double *mult;     // 2 x [mmax][UPD_MS] (negated) multipliers of the current / next panel
  double *dpre;     // 2 x [NB][CH_DPS]  pre-updated diagonal block of the current / next panel
  int msz;          // doubles per multiplier table
  double *dg;       // [NB][UPD_DS]  diagonal block of the current panel (factor scratch)
  double *Wm;       // [NB][UPD_WS]  W = U_pp^-T of the current panel
  double *pan;      // panel buffer [NB][panw]
  int panw;
};
__host__ __device__ inline size_t chol_smem_doubles(int kmax) {
  const size_t mmax = 2 * upd_keven(kmax);
  return 2 * mmax * UPD_MS + 2 * UPD_NB * CH_DPS + UPD_NB * UPD_DS + UPD_NB * UPD_WS + upd_pan_doubles(kmax);
}
__device__ __forceinline__ CholSmem chol_carve(uint8_t *base, int kmax) {
  CholSmem u;
  const int mmax = 2 * upd_keven(kmax);
  double *p = reinterpret_cast<double *>(base);
  u.msz = mmax * UPD_MS;
  u.mult = p;  p += (size_t)2 * u.msz;
  u.dpre = p;  p += 2 * UPD_NB * CH_DPS;
  u.dg = p;  p += UPD_NB * UPD_DS;
  u.Wm = p;  p += UPD_NB * UPD_WS;
  u.pan = p;
  u.panw = upd_panw(kmax);
  return u;
}

__global__ void __launch_bounds__(UPD_THREADS, 2) upd_chol_kernel(const Sl2Dev d, int stream_lo) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  pdl_prologue();
  const CholSmem sm = chol_carve(smem_raw, d.kmax);
  const int s = stream_lo + blockIdx.x;
  const int tid = threadIdx.x;
  const int ldg = d.ldg;
  double *__restrict__ G = d.G + (size_t)s * d.mmax * ldg;
  double *__restrict__ Wp = d.Wp + (size_t)s * SL2_MAX_PANELS * 256;
  const int warp = tid >> 5, lane = tid & 31;
  const int lr = lane >> 2, lc = lane & 3;  // DMMA fragment coordinates
  __shared__ int s_next;
  const int m = d.upd_m[s];
  if (m == 0) return;
  const int width = m;
  const int PW = sm.panw;
  if (tid == 0) s_next = 1;  // item 0 is reserved for warp 0
  __syncthreads();

  for (int i0 = 0, pidx = 0; i0 < m; i0 += UPD_NB, ++pidx) {
    // (offsets from the carved bases, not a table of pointers: the accesses stay shared-memory instructions)
    const int par = pidx & 1;
    const double *__restrict__ mcur = sm.mult + par * sm.msz;
    double *__restrict__ mnext = sm.mult + (par ^ 1) * sm.msz;
    const double *__restrict__ dcur = sm.dpre + par * (UPD_NB * CH_DPS);
    double *__restrict__ dnext = sm.dpre + (par ^ 1) * (UPD_NB * CH_DPS);
    const int nbp = min(UPD_NB, m - i0);
    const int n0 = i0 + UPD_NB;                       // next panel
    const int nbn = n0 < m ? min(UPD_NB, m - n0) : 0;
    const int ngroups = (width - i0 + 7) >> 3;
    const int nk = i0 >> 2;  // k-steps of 4 finished rows; i0 is a multiple of 16
    // 8-column groups per batch item: about one item per warp (7 warps besides the one that factors)
    const int gb = 4;
    const int nbatch = ngroups > 2 ? (ngroups - 2 + gb - 1) / gb : 0;
    const int nitems = 2 + nbatch;
    bool first = true;
    for (;;) {
      int it;
      if (warp == 0 && first) {
        it = 0;
      } else {
        if (lane == 0) it = atomicAdd(&s_next, 1);
        it = __shfl_sync(0xffffffffu, it, 0);
      }
      if (it >= nitems) break;
      if (it == 0) {
        // ---- diagonal block of this panel: pre-updated block minus panel p-1's rows, then factor ----------
        first = false;
        double c[2][4];  // [column group q][2 M tile mt + element]
        if (pidx == 0) {
#pragma unroll
          for (int q = 0; q < 2; ++q)
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
              const int r = mt * 8 + lr, cc = 8 * q + 2 * lc;
              c[q][2 * mt] = (r < nbp && cc < width) ? G[(size_t)r * ldg + cc] : 0.0;
              c[q][2 * mt + 1] = (r < nbp && cc + 1 < width) ? G[(size_t)r * ldg + cc + 1] : 0.0;
            }
        } else {
#pragma unroll
          for (int q = 0; q < 2; ++q)
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
              const double2 v = *reinterpret_cast<const double2 *>(dcur + (mt * 8 + lr) * CH_DPS + 8 * q + 2 * lc);
              c[q][2 * mt] = v.x;
              c[q][2 * mt + 1] = v.y;
            }
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const int st = nk - 4 + u;
            const double a[2] = {mcur[(4 * st + lc) * UPD_MS + lr], mcur[(4 * st + lc) * UPD_MS + 8 + lr]};
            dmma1684(c[0], a, -a[0]);
            dmma1684(c[1], a, -a[1]);
          }
        }
        // Factor the 16x16 diagonal block and form W = U_pp^-T (the panel is then finished with one
        // more DMMA product U_panel = W * C_panel).  This is the serial path of the panel, so it is
        // kept short: two 8x8 register/shuffle factorizations (chol8_inv) and 8x8 DMMA products
        //   U12 = W11 A12,  A22 -= U12^T U12,  W21 = -W22 (U12^T W11)
        // on the block in its own scratch (identity padding for the ragged last panel).
        {
          double *dg = sm.dg;
#pragma unroll
          for (int q = 0; q < 2; ++q)
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
              const int r = mt * 8 + lr, cc = 8 * q + 2 * lc;
              const bool rv = r < nbp;
              *reinterpret_cast<double2 *>(dg + r * UPD_DS + cc) =
                  make_double2((rv && cc < nbp) ? c[q][2 * mt] : (r == cc ? 1.0 : 0.0),
                               (rv && cc + 1 < nbp) ? c[q][2 * mt + 1] : (r == cc + 1 ? 1.0 : 0.0));
            }
          // W12 = 0 (the two diagonal blocks of W are written whole by chol8_inv, W21 by the glue below)
          sm.Wm[(lane >> 3) * UPD_WS + 8 + (lane & 7)] = 0.0;
          sm.Wm[(4 + (lane >> 3)) * UPD_WS + 8 + (lane & 7)] = 0.0;
          __syncwarp();
          chol8_inv(dg, sm.Wm, 0, lane);
          __syncwarp();
          {  // U12 = W11 * A12
            double c0 = 0.0, c1 = 0.0;
#pragma unroll
            for (int ks = 0; ks < 2; ++ks)
              dmma884(c0, c1, sm.Wm[lr * UPD_WS + 4 * ks + lc], dg[(4 * ks + lc) * UPD_DS + 8 + lr]);
            __syncwarp();
            *reinterpret_cast<double2 *>(dg + lr * UPD_DS + 8 + 2 * lc) = make_double2(c0, c1);
          }
          __syncwarp();
          {  // A22 -= U12^T U12   (A(i,k) = U12(k,i) and B(k,n) = U12(k,n): the same fragment)
            double2 cv = *reinterpret_cast<const double2 *>(dg + (8 + lr) * UPD_DS + 8 + 2 * lc);
#pragma unroll
            for (int ks = 0; ks < 2; ++ks) {
              const double v = dg[(4 * ks + lc) * UPD_DS + 8 + lr];
              dmma884(cv.x, cv.y, -v, v);
            }
            *reinterpret_cast<double2 *>(dg + (8 + lr) * UPD_DS + 8 + 2 * lc) = cv;
          }
          __syncwarp();
          chol8_inv(dg, sm.Wm, 8, lane);
          __syncwarp();
          {  // T = U12^T W11 (parked in the unused lower-left block of dg), W21 = -W22 T
            double t0 = 0.0, t1 = 0.0;
#pragma unroll
            for (int ks = 0; ks < 2; ++ks)
              dmma884(t0, t1, dg[(4 * ks + lc) * UPD_DS + 8 + lr], sm.Wm[(4 * ks + lc) * UPD_WS + lr]);
            *reinterpret_cast<double2 *>(dg + (8 + lr) * UPD_DS + 2 * lc) = make_double2(t0, t1);
            __syncwarp();
            double w0 = 0.0, w1 = 0.0;
#pragma unroll
            for (int ks = 0; ks < 2; ++ks)
              dmma884(w0, w1, -sm.Wm[(8 + lr) * UPD_WS + 8 + 4 * ks + lc], dg[(8 + 4 * ks + lc) * UPD_DS + lr]);
            *reinterpret_cast<double2 *>(sm.Wm + (8 + lr) * UPD_WS + 2 * lc) = make_double2(w0, w1);
          }
          __syncwarp();
          if (nbp < UPD_NB)  // ragged last panel: rows / columns of the padding carry no W
            for (int e = lane; e < UPD_NB * UPD_NB; e += 32) {
              const int i = e >> 4, j = e & 15;
              if (i >= nbp || j >= nbp) sm.Wm[i * UPD_WS + j] = 0.0;
            }
        }
      } else if (it == 1) {
        // ---- look-ahead: diagonal block of panel p+1 minus the contributions of rows < i0 -----------------
        if (nbn == 0) continue;
        double c[2][4];  // starts from the S entries of the block (their load overlaps the first B loads)
#pragma unroll
        for (int q = 0; q < 2; ++q)
#pragma unroll
          for (int mt = 0; mt < 2; ++mt) {
            const int r = mt * 8 + lr, cc = 8 * q + 2 * lc;
            c[q][2 * mt] = (r < nbn && n0 + cc < width) ? G[(size_t)(n0 + r) * ldg + n0 + cc] : 0.0;
            c[q][2 * mt + 1] = (r < nbn && n0 + cc + 1 < width) ? G[(size_t)(n0 + r) * ldg + n0 + cc + 1] : 0.0;
          }
        double v[CH_D][2];
        const size_t kstride = (size_t)4 * ldg;
        const double *gpre = G + (size_t)lc * ldg + n0 + lr;  // next k-step to request
        double *mp = mnext + lc * UPD_MS + lr;               // where the multipliers of the next k-step to use go
        const bool v0 = lr < nbn, v1 = 8 + lr < nbn;         // rows of the (ragged) next panel
        auto loadv = [&](double *dst) {  // negated multipliers U(k, n0 + r) of the next panel
          const double x0 = gpre[0], x1 = gpre[8];
          dst[0] = v0 ? -x0 : 0.0;
          dst[1] = v1 ? -x1 : 0.0;
          gpre += kstride;
        };
        auto step = [&](const double *vu) {
          const double a[2] = {vu[0], vu[1]};
          mp[0] = a[0];
          mp[8] = a[1];
          mp += 4 * UPD_MS;
          dmma1684(c[0], a, -a[0]);
          dmma1684(c[1], a, -a[1]);
        };
#pragma unroll
        for (int u = 0; u < CH_D - 1; ++u)
          if (u < nk) loadv(v[u]);
        int kb = 0;
        for (; kb + CH_D <= nk; kb += CH_D) {
#pragma unroll
          for (int u = 0; u < CH_D; ++u) {
            if (kb + u + CH_D - 1 < nk) loadv(v[(u + CH_D - 1) % CH_D]);  // warp-uniform
            step(v[u]);
          }
        }
#pragma unroll
        for (int q = 0; q < 2; ++q)
#pragma unroll
          for (int mt = 0; mt < 2; ++mt)
            *reinterpret_cast<double2 *>(dnext + (mt * 8 + lr) * CH_DPS + 8 * q + 2 * lc) =
                make_double2(c[q][2 * mt], c[q][2 * mt + 1]);
      } else {
        // ---- trailing columns of this panel: C(16 x cols) - A(16 x i0) * B(i0 x cols) ---------------------
        // few column groups left (late panels): narrow items with a deep B pipeline, so that every warp has an
        // item and an item's nk dependent k-steps do not each wait for L2
        const int bt = it - 2;
        if (gb == 4) chol_batch<4, 4>(G, ldg, mcur, sm.pan, PW, i0, nbp, nk, ngroups, width, 2 + bt * 4, lr, lc);
        else if (gb == 2) chol_batch<2, 8>(G, ldg, mcur, sm.pan, PW, i0, nbp, nk, ngroups, width, 2 + bt * 2, lr, lc);
        else chol_batch<1, 8>(G, ldg, mcur, sm.pan, PW, i0, nbp, nk, ngroups, width, 2 + bt, lr, lc);
      }
    }
    __syncthreads();
    // finish the panel: rows of U for the 16 diagonal columns, U_panel = W * C_panel (DMMA) for
    // all other columns, written straight to G from the C fragments; W_pp goes to the solve kernel
    const int ncol = width - i0;
    for (int e = tid; e < UPD_NB * UPD_NB; e += UPD_THREADS) {
      const int r = e / UPD_NB, cc = e - r * UPD_NB;
      if (r < nbp && cc < nbp && i0 + cc < width)
        G[(size_t)(i0 + r) * ldg + i0 + cc] = (cc >= r) ? sm.dg[r * UPD_DS + cc] : 0.0;
      Wp[(size_t)pidx * 256 + e] = sm.Wm[r * UPD_WS + cc];
      // multipliers of the next panel from this panel's rows: the entries the DMMA loop below does not write
      if (r >= nbp || UPD_NB + cc >= ncol) mnext[(i0 + r) * UPD_MS + cc] = 0.0;
    }
    if (tid == 0) s_next = 1;
    {
      double aw[4][2];  // m16n8k4 A fragments of W, k-step ks
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) aw[ks][mt] = sm.Wm[(mt * 8 + lr) * UPD_WS + 4 * ks + lc];
      // FG column groups per iteration: independent DMMA chains.  Only full panels reach this loop
      // with columns to do (a ragged last panel has ncol == nbp: nothing right of the diagonal block).
      constexpr int FG = 4;
      for (int gb = 2 + warp; gb * 8 < ncol; gb += FG * (UPD_THREADS / 32)) {
        double c[FG][4];  // c[f][2 mt + e]: row 8 mt + lr
#pragma unroll
        for (int f = 0; f < FG; ++f) c[f][0] = c[f][1] = c[f][2] = c[f][3] = 0.0;
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
          double bv[FG];
#pragma unroll
          for (int f = 0; f < FG; ++f) {
            const int cb = (gb + f * (UPD_THREADS / 32)) * 8 + lr;
            bv[f] = cb < ncol ? sm.pan[(size_t)(4 * ks + lc) * PW + cb] : 0.0;
          }
#pragma unroll
          for (int f = 0; f < FG; ++f) dmma1684(c[f], aw[ks], bv[f]);
        }
#pragma unroll
        for (int f = 0; f < FG; ++f) {
          const int gq = gb + f * (UPD_THREADS / 32);
          const int cc = gq * 8 + 2 * lc;
#pragma unroll
          for (int mt = 0; mt < 2; ++mt) {
            const int r = mt * 8 + lr;
            if (r < nbp && cc < ncol) {
              double *dst = G + (size_t)(i0 + r) * ldg + i0 + cc;
              if (cc + 1 < ncol) *reinterpret_cast<double2 *>(dst) = make_double2(c[f][2 * mt], c[f][2 * mt + 1]);
              else *dst = c[f][2 * mt];
              if (gq < 4) {  // columns of the next panel's diagonal block: its multipliers for these rows
                mnext[(i0 + r) * UPD_MS + cc - UPD_NB] = -c[f][2 * mt];
                if (cc + 1 < ncol) mnext[(i0 + r) * UPD_MS + cc + 1 - UPD_NB] = -c[f][2 * mt + 1];
              }
            }
          }
        }
      }
    }
    __syncthreads();
  }
}

// =============================================================================================
// kernel 2: upd_solve — Y = U^-T [H P | nu], 8 columns per warp held in registers
// =============================================================================================
// C fragments of a 16-row block (two M tiles: c[mt][e] = X(8 mt + lane/4, 2 (lane%4) + e)) -> B fragment of
// its k-step ks (rows 4 ks .. 4 ks + 3): lane (lr, lc) receives X(4 ks + lc, lr).
__device__ __forceinline__ double c_to_b(const double (&c)[2][2], int ks, int lane) {
  const int lr = lane >> 2, lc = lane & 3;
  const int src = ((4 * (ks & 1) + lc) << 2) | (lr >> 1);
  const double v0 = __shfl_sync(0xffffffffu, c[ks >> 1][0], src);
  const double v1 = __shfl_sync(0xffffffffu, c[ks >> 1][1], src);
  return (lr & 1) ? v1 : v0;
}

// NP = number of 16-row panels the instantiation covers (m <= 16 NP).  Column c of the slab space is
// column m + c of G: c < n is H P, c == n is nu.
//
// Right-looking, everything in registers: the warp holds all rows of its 8 columns as DMMA ACCUMULATORS
// (C layout: tile j = rows 8j..8j+7).  Per panel p: Y_p = W_pp C_p (8 DMMAs, C_p moved to the B layout by
// shuffles), the finished rows go straight to G as 16-byte stores, and every later row tile j gets
// acc_j -= U(panel, tile j)^T Y_p: 4 m16n8k4 DMMAs per pair of the warp's tiles (k-step outer, pair inner:
// consecutive DMMAs never share an accumulator), A from the panel's rows of U in shared memory, B = Y_p from
// registers.  On an H100 the 16-row FP64 MMA shapes run at about 1.5x the rate of m8n8k4 (tools/dmma_rate.cu).
// Staging: ALL panels of U (the part right of the diagonal blocks, <= 166 KB at m = 208) and all W_pp are
// requested up front by warp 0 as bulk copies (one instruction per 16-row x row-segment / per W row, completion
// counted in bytes on one mbarrier per panel), so the only latency the kernel ever waits for is the first
// panel's, nobody computes a staging address, and there is NO CTA-wide barrier in the panel loop: a warp waits
// on the mbarrier of the panel it needs and otherwise runs at its own pace.  (Measured before: a 2-deep cp.async
// ring left the late, small panels bound by the L2 round trip of their own staging, and staging everything with
// per-thread cp.async cost a large share of the kernel in index arithmetic.)  NP = 16 does not fit one SM that way: its
// panels >= SPLIT are requested at panel REUSE into the space of panels 0..REUSE-1 (one CTA barrier).
template <int NP> struct SolveLayout {
  static constexpr int SPLIT = NP > 13 ? 6 : NP;   // panels >= SPLIT are staged late (second generation)
  static constexpr int REUSE = NP > 13 ? 4 : NP;   // ... once panels < REUSE have been consumed
  __host__ __device__ static constexpr int pw(int p) { return 16 * (NP - 1 - p) + 4; }  // row stride (= 4 mod 16)
  __host__ __device__ static constexpr int off_lin(int p0, int p) {  // doubles before panel p when packing starts at p0
    int o = 0;
    for (int q = p0; q < p; ++q) o += 16 * pw(q);
    return o;
  }
  __host__ __device__ static constexpr int off(int p) { return p < SPLIT ? off_lin(0, p) : off_lin(SPLIT, p); }
  static constexpr int PAN_DOUBLES = off_lin(0, SPLIT < NP - 1 ? SPLIT : NP - 1);
  static constexpr int SMEM_DOUBLES = PAN_DOUBLES + NP * 16 * UPD_WS + NP + (NP & 1) +  // one mbarrier per panel
                                      2 * SOLVE_MAX_WARPS * 2 * 32 * 2 +    // C-tile exchange of the warp pairs
                                      SOLVE_MAX_WARPS * 128;                // Y_p exchange
  static_assert(SPLIT == NP || off_lin(SPLIT, NP - 1) <= off_lin(0, REUSE), "second generation must fit");
};

// Two warps share a group of 8 columns: warp (g, rho) owns the row tiles j = 2t + rho, so a thread keeps NP
// tiles (not 2 NP) and 16 warps fit one SM -- 4 per scheduler instead of 2, which is what hides the shared-memory
// latency in front of every DMMA (8 warps x 228 registers left the FP64 pipe mostly idle).  Per panel the
// two warps swap their C tile through shared memory (one named barrier of 64 threads), each forms ITS M tile of
// Y_p = W_pp C_p (4 DMMAs), stores it, and the pair swaps the two tiles of Y_p through shared memory as well (a second
// 64-thread barrier; the B fragments of Y_p are then plain shared loads).  (Until the middle of round 2 both warps
// formed all of Y_p -- 8 DMMAs, 4 of them redundant, fragments moved by 8 shuffles: measured slower.)
//
// FULL: when the measurement rows reach into the last panel the instantiation covers (m > 16 NP - 16: the benchmark
// shapes), every row tile of every panel exists except possibly the very last one, whose staged columns are zero-filled
// instead -- so the trailing update needs NO per-tile predicate.  (With the predicate the compiler wraps every DMMA
// in @P WARPSYNC / NOP / ISETP and keeps the predicates in a spilled mask: ~6 instructions per DMMA.)
template <int NP>
__global__ void __launch_bounds__(64 * SOLVE_MAX_WARPS, 1) upd_solve_kernel(const Sl2Dev d, int stream_lo) {
  using L = SolveLayout<NP>;
  extern __shared__ __align__(16) uint8_t smem_raw[];
  pdl_prologue();
  double *pan = reinterpret_cast<double *>(smem_raw);  // panel p at L::off(p): [16][L::pw(p)]  U(16p + r, 16p + 16 + c)
  double *Wm = pan + L::PAN_DOUBLES;                   // [NP][16][UPD_WS]
  const uint32_t bars = smem_u32(Wm + NP * 16 * UPD_WS);  // [NP] mbarriers
  double2 *xbuf = reinterpret_cast<double2 *>(Wm + NP * 16 * UPD_WS + NP + (NP & 1));  // [2][groups][2][32]
  double *ybuf = reinterpret_cast<double *>(xbuf + 2 * SOLVE_MAX_WARPS * 2 * 32);       // [groups][16][8]  Y_p
  const int s = stream_lo + blockIdx.y;
  const int m = d.upd_m[s];
  if (m == 0) return;
  const int tid = threadIdx.x, nthr = blockDim.x;
  const int ngrp = nthr >> 6;  // column groups of this CTA
  const int warp = tid >> 5, lane = tid & 31, lr = lane >> 2, lc = lane & 3;
  const int g = warp % ngrp, rho = warp / ngrp;
  const int n = SL2_NXV + 3 * d.nfeat[s];
  const int ncols = n + 1;
  if (blockIdx.x * ngrp * 8 >= ncols) return;  // whole CTA beyond the last column
  const int ldg = d.ldg;
  double *__restrict__ G = d.G + (size_t)s * d.mmax * ldg;
  const double *__restrict__ Wp = d.Wp + (size_t)s * SL2_MAX_PANELS * 256;
  const int m8 = (m + 7) & ~7;
  const bool full = L::SPLIT == NP && m8 >= 16 * NP - 8;  // uniform over the CTA
  const int zend = full ? 16 * NP : m8;

  if (tid == 0) {
    for (int p = 0; p < NP; ++p) mbar_init(bars + 8 * p, 1);
    fence_barrier_init();
    fence_proxy_async();
  }
  // the columns m .. zend-1 of a staged panel are read (rows of the last tile(s) that do not exist) but not copied
  auto zero_pads = [&](int plo, int phi) {
    for (int e = tid; e < (phi - plo) * 16; e += nthr) {
      const int p = plo + (e >> 4), r = e & 15;
      const int cfirst = 16 * p + 16;
      if (16 * p < m)
        for (int c = max(m, cfirst); c < zend; ++c) pan[L::off(p) + r * L::pw(p) + (c - cfirst)] = 0.0;
    }
  };
  zero_pads(0, L::SPLIT);
  __syncthreads();
  // warp 0: lane r < 16 requests row r of U(panel p) right of the diagonal block, lane 16 + r row r of W_pp
  auto request = [&](int p) {
    if (16 * p < m) {
      const int cfirst = 16 * p + 16;
      const int nrow = min(16, m - 16 * p);
      const uint32_t ubytes = m > cfirst ? (uint32_t)(m - cfirst) * 8u : 0u;
      const uint32_t bar = bars + 8 * p;
      if (lane == 0) mbar_expect_tx(bar, (uint32_t)nrow * ubytes + 16u * 128u);
      __syncwarp();
      if (lane < 16) {
        if (lane < nrow && ubytes)
          bulk_g2s(pan + L::off(p) + lane * L::pw(p), G + (size_t)(16 * p + lane) * ldg + cfirst, ubytes, bar);
      } else {
        bulk_g2s(Wm + ((size_t)p * 16 + (lane - 16)) * UPD_WS, Wp + (size_t)p * 256 + (lane - 16) * 16, 128u, bar);
      }
    }
  };
  if (warp == 0) {
#pragma unroll 1
    for (int p = 0; p < L::SPLIT; ++p) request(p);
  }

  int xpar = 0;
  // one group of 8 columns through all panels; FULL (compile time): no tile / panel predicates
  auto solve_group = [&](auto full_c, const int grp) {
    constexpr bool FULL = decltype(full_c)::value;
    const int c0 = 8 * grp;        // first column of this warp pair
    const bool wact = c0 < ncols;  // warp pairs past the last column have nothing to do
    const int cc = c0 + 2 * lc;    // this lane's two columns (C layout)
    const int cval = wact ? min(2, ncols - cc) : 0;  // how many of them exist (<= 0: none)
    double *gcol = G + m + cc;
    double acc[(NP + 1) & ~1][2];  // tile j = 2 t + rho: rows 8 j + lr, columns cc, cc + 1 (acc[NP]: zero pad)
    {  // the next group's tiles: towards L2 now (H P is larger than L2 at the benchmark's stream count; the registers are all taken)
      const int ccn = cc + 8 * (int)(gridDim.x * ngrp);
      if (L::SPLIT >= NP && ccn < ncols) {
#pragma unroll
        for (int t = 0; t < NP; ++t) {
          const int row = 8 * (2 * t + rho) + lr;
          if (row < m) asm volatile("prefetch.global.L2 [%0];" ::"l"(G + m + ccn + (size_t)row * ldg));
        }
      }
    }
#pragma unroll
    for (int t = 0; t < ((NP + 1) & ~1); ++t) {
      const int row = 8 * (2 * t + rho) + lr;
      acc[t][0] = acc[t][1] = 0.0;
      if (row < m) {
        if (cval >= 2) {
          const double2 v = *reinterpret_cast<const double2 *>(gcol + (size_t)row * ldg);
          acc[t][0] = v.x;
          acc[t][1] = v.y;
        } else if (cval == 1) {
          acc[t][0] = gcol[(size_t)row * ldg];
        }
      }
    }

#pragma unroll
    for (int p = 0; p < NP; ++p) {
      if (FULL || 16 * p < m) {  // uniform over the CTA
        if (L::SPLIT < NP && p == L::REUSE) {
          __syncthreads();  // every warp is done with panels < REUSE: their space takes the second generation
          zero_pads(L::SPLIT, NP);
          __syncthreads();
          if (warp == 0) {
            fence_proxy_async();  // generic-proxy reads of the old panels are ordered before the bulk writes
#pragma unroll 1
            for (int q = L::SPLIT; q < NP; ++q) request(q);
          }
        }
        if (!wact) continue;
        // swap the C tiles of panel p with the partner warp
        xpar ^= 1;  // alternates over every panel this pair executes (also across column groups)
        double2 *xb = xbuf + ((size_t)(xpar * ngrp + g) * 2) * 32;
        xb[rho * 32 + lane] = make_double2(acc[p][0], acc[p][1]);
        asm volatile("bar.sync %0, 64;" ::"r"(1 + g) : "memory");
        const double2 other = xb[(rho ^ 1) * 32 + lane];
        const double cp2[2][2] = {{rho ? other.x : acc[p][0], rho ? other.y : acc[p][1]},
                                  {rho ? acc[p][0] : other.x, rho ? acc[p][1] : other.y}};
        mbar_wait(bars + 8 * p, 0);
        const double *pb = pan + L::off(p);
        const int PW = L::pw(p);
        const double *wb = Wm + (size_t)p * 16 * UPD_WS;
        // this warp's M tile of Y_p = W_pp * C_p: rows 8 rho .. 8 rho + 7
        double cb[4];
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) cb[ks] = c_to_b(cp2, ks, lane);
        double d0 = 0.0, d1 = 0.0;
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) dmma884(d0, d1, wb[(8 * rho + lr) * UPD_WS + 4 * ks + lc], cb[ks]);
        {  // the finished rows: 16-byte stores from the C fragments
          const int row = 16 * p + 8 * rho + lr;
          if (row < m) {
            if (cval >= 2) *reinterpret_cast<double2 *>(gcol + (size_t)row * ldg) = make_double2(d0, d1);
            else if (cval == 1) gcol[(size_t)row * ldg] = d0;
          }
        }
        if (p + 1 < NP) {
          // both tiles through shared memory, row-major [16][8]: the B fragment of k-step ks is Y_p(4 ks + lc, lr).
          // (No second buffer: the partner passes the C-tile barrier of the next panel only after these loads.)
          double *yg = ybuf + (size_t)g * 128;
          *reinterpret_cast<double2 *>(yg + (8 * rho + lr) * 8 + 2 * lc) = make_double2(d0, d1);
          asm volatile("bar.sync %0, 64;" ::"r"(1 + g) : "memory");
          double yb[4];
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) yb[ks] = -yg[(4 * ks + lc) * 8 + lr];
          // this warp's later row tiles: acc_j -= U(panel, tile j)^T Y_p as m16n8k4 products over the fixed pairs
          // of its tiles (2u, 2u + 1): the pair's rows are the two halves of M, so the accumulators of a pair stay
          // in one register quad for every panel (k-step outer, pair inner: consecutive DMMAs never share an
          // accumulator).  A tile that is finished (<= p), past the last one or, without FULL, past m8 (its columns
          // are not staged) gets zero rows of A.
          const double *pbr = pb + 8 * rho + lr;
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
            for (int t = (p + 1) & ~1; t < NP; t += 2) {
              const bool has[2] = {t > p && (FULL || 8 * (2 * t + rho) < m),
                                   t + 1 < NP && (FULL || 8 * (2 * t + 2 + rho) < m)};  // warp-uniform
              if (has[0] || has[1]) {
                double a[2];
#pragma unroll
                for (int h = 0; h < 2; ++h) a[h] = has[h] ? pbr[(4 * ks + lc) * PW + 16 * (t + h - p - 1)] : 0.0;
                double c[4] = {acc[t][0], acc[t][1], acc[t + 1][0], acc[t + 1][1]};
                dmma1684(c, a, yb[ks]);
                acc[t][0] = c[0];
                acc[t][1] = c[1];
                acc[t + 1][0] = c[2];
                acc[t + 1][1] = c[3];
              }
            }
          }
        }
      }
    }
  };
  // The warp pair walks the column groups g, g + gridDim.x * ngrp, ...: with one CTA per stream (the batched
  // launch) U is staged ONCE for all of the stream's columns and the pairs drift apart, so one pair's reload of
  // its accumulators hides behind the other pairs' DMMAs; nothing below synchronises the CTA (NP <= 13).
  for (int grp = blockIdx.x * ngrp + g; L::SPLIT < NP ? grp == (int)(blockIdx.x * ngrp + g) : 8 * grp < ncols;
       grp += gridDim.x * ngrp) {
    if (L::SPLIT == NP && full) solve_group(std::true_type{}, grp);
    else solve_group(std::false_type{}, grp);
  }
}

// =============================================================================================
// kernel 3: upd_syrk — P -= Y^T Y on 64x64 tiles, x += Y^T w from the column that carries nu
// =============================================================================================
// One 64x64 tile T = sum_{k < m} A(k, :)^T B(k, :) per CTA, A / B = 64-column slabs of Y (rows of G, row stride
// ldg) at columns m + 64 ta / m + 64 tb; a diagonal tile stages one slab and reads it twice.  FP64 DMMA tiles;
// the slabs are staged by cp.async (LDGSTS) in chunks of KC rows into a ring of ST conflict-free (stride UPD_YS)
// stages, one __syncthreads per chunk: the stage refilled after the barrier of chunk c is the one chunk c-1 was
// read from.
// Columns >= n + 1 and rows >= m are zero-filled.
// Four warps, each a 32x32 quarter of the tile as 2 x 4 m16n8k8 products per 8-row k-step: per k-row a warp reads
// 64 doubles of the slabs for 1024 FMAs (0.5 B of shared memory per FMA) and the fill writes 0.25 B per FMA more.
// The 16x32 warp tiles of 8 warps this replaced read 0.75 B per FMA, which with the fill is the 1 B per FMA an
// H100 SM's shared memory delivers at its FP64 tensor rate (128 B and 128 FMA per clock).
// Warp w owns rows 32*(w%2).. and columns 32*(w/2).. of the tile:
//   acc[i][j][e] = T(32*(w%2) + 16*i + 8*(e/2) + lane/4, 32*(w/2) + 8*j + 2*(lane%4) + e%2).
constexpr int SYRK_THREADS = 128;
template <int KC, int ST>
__global__ void __launch_bounds__(SYRK_THREADS, 3) upd_syrk_kernel(const Sl2Dev d, int stream_lo) {
  constexpr int STAGE = 2 * KC * UPD_YS;  // doubles per stage (A slab, B slab)
  constexpr int NW = SYRK_THREADS / 32;
  extern __shared__ __align__(16) uint8_t smem_raw[];
  double *stage_buf = reinterpret_cast<double *>(smem_raw);
  pdl_prologue();
  const int s = stream_lo + blockIdx.y;
  const int m = d.upd_m[s];
  if (m == 0) return;
  const int n = SL2_NXV + 3 * d.nfeat[s];
  // tiles in (tb outer, ta <= tb inner) order
  int tb = 0;
  const int t = blockIdx.x;
  while ((tb + 1) * (tb + 2) / 2 <= t) ++tb;
  const int ta = t - tb * (tb + 1) / 2;
  if (tb * 64 >= n + 1) return;  // this stream's map is smaller than the capacity the grid was sized for
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, lr = lane >> 2, lc = lane & 3;
  const int wa = (warp & 1) * 32, wb = (warp >> 1) * 32;
  const int ld = d.ld, ldg = d.ldg;
  double *__restrict__ P = d.P + (size_t)s * ld * ld;
  double *__restrict__ x = d.x + (size_t)s * ld;
  const double *__restrict__ G = d.G + (size_t)s * d.mmax * ldg;
  const bool diag = ta == tb;
  // 8x8 blocks of the warp's 32 x 32 sub-tile (bit 4 bi + bj = block (bi, bj)): an off-diagonal tile computes all of
  // them and mirrors every one; a diagonal tile writes the blocks on / above the diagonal and mirrors the ones strictly
  // above.  A diagonal warp issues the 6 of its 8 products that hold such a block (product (i, j) holds blocks
  // (2i, j) and (2i+1, j)); the warp below the diagonal issues none.  The shapes are compiled as separate loop
  // bodies chosen per warp, with no predicate per DMMA.
  const int bi0 = wa >> 3, bj0 = wb >> 3;
  unsigned cmask = 0xFFFFu, mmask = 0xFFFFu;
  if (diag) {
    cmask = mmask = 0u;
#pragma unroll
    for (int bi = 0; bi < 4; ++bi)
#pragma unroll
      for (int bj = 0; bj < 4; ++bj) {
        if (bi0 + bi <= bj0 + bj) cmask |= 1u << (4 * bi + bj);
        if (bi0 + bi < bj0 + bj) mmask |= 1u << (4 * bi + bj);
      }
  }
  const bool skip = cmask == 0u;  // sub-tile strictly below the diagonal: mirrored instead
  // the tile of P this warp updates: into L2 while the products run (the epilogue reads it once)
  if (!skip) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int a = ta * 64 + wa + i * 8, bq = tb * 64 + wb + lane;
      if (a < n && bq < n) asm volatile("prefetch.global.L2 [%0];" ::"l"(P + a + (size_t)ld * bq));
    }
  }
  const int kr = m, lim = m + n + 1;
  const int nchunk = (kr + KC - 1) / KC;
  const int cA = m + ta * 64 + 2 * lane, cB = m + tb * 64 + 2 * lane;
  const int bytesA = cA + 1 < lim ? 16 : (cA < lim ? 8 : 0);
  const int bytesB = cB + 1 < lim ? 16 : (cB < lim ? 8 : 0);
  const double *srcA = G + (bytesA ? cA : 0);
  const double *srcB = G + (bytesB ? cB : 0);
  // stage loader: 2 slabs x KC rows x 64 columns; thread = (row warp + NW*j, 16-byte segment `lane`).  Chunks are
  // staged in increasing order, so the source pointers just advance; a full chunk costs the copies, two pointer
  // bumps and nothing else.
  const double *pa = srcA + (size_t)warp * ldg, *pb = srcB + (size_t)warp * ldg;  // row `warp` of the next chunk
  const uint32_t sdst = smem_u32(stage_buf + 2 * lane + warp * UPD_YS);
  const size_t rstep = (size_t)NW * ldg;
  auto stage = [&](int chunk) {
    const uint32_t dd = sdst + (uint32_t)(chunk % ST) * (STAGE * 8);
    if ((chunk + 1) * KC <= kr) {  // every row of the chunk exists (CTA-uniform)
#pragma unroll
      for (int j = 0; j < KC / NW; ++j) {
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dd + j * NW * UPD_YS * 8),
                     "l"(pa + j * rstep), "r"(bytesA)
                     : "memory");
        if (!diag)
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dd + (KC + j * NW) * UPD_YS * 8),
                       "l"(pb + j * rstep), "r"(bytesB)
                       : "memory");
      }
    } else {  // the ragged last chunk: rows past kr are zero-filled
#pragma unroll
      for (int j = 0; j < KC / NW; ++j) {
        const bool kv = chunk * KC + warp + NW * j < kr;
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dd + j * NW * UPD_YS * 8),
                     "l"(kv ? pa + j * rstep : srcA), "r"(kv ? bytesA : 0)
                     : "memory");
        if (!diag)
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dd + (KC + j * NW) * UPD_YS * 8),
                       "l"(kv ? pb + j * rstep : srcB), "r"(kv ? bytesB : 0)
                       : "memory");
      }
    }
    pa += (size_t)KC * ldg;
    pb += (size_t)KC * ldg;
  };
  double acc[2][4][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.0;
#pragma unroll
  for (int c = 0; c < ST - 1; ++c) {
    if (c < nchunk) stage(c);
    cp_async_commit();
  }
  for (int ch = 0; ch < nchunk; ++ch) {
    cp_async_wait<ST - 2>();  // chunk ch has landed (one group is committed per iteration, empty or not)
    __syncthreads();          // ... for every thread's part of it, and chunk ch-1 has been read by every warp
    if (ch + ST - 1 < nchunk) stage(ch + ST - 1);
    cp_async_commit();
    if (!skip) {
      const double *Ya = stage_buf + (size_t)(ch % ST) * STAGE;
      const double *Yb = diag ? Ya : Ya + KC * UPD_YS;
      const int krem = kr - ch * KC;  // rows of this chunk that exist (the rest, to the chunk's end, is zero fill)
      auto chunk = [&](auto diag_c) {
        constexpr bool DIAG = decltype(diag_c)::value;  // products (1, 0) and (1, 1) lie below the diagonal
        auto kstep = [&](int kk) {
          double a[2][4], b[4][2];
#pragma unroll
          for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int e = 0; e < 4; ++e)
              a[i][e] = Ya[(kk + lc + 4 * (e >> 1)) * UPD_YS + wa + 16 * i + 8 * (e & 1) + lr];
#pragma unroll
          for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) b[j][e] = Yb[(kk + lc + 4 * e) * UPD_YS + wb + j * 8 + lr];
#pragma unroll
          for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j)
              if (!DIAG || 2 * i <= j) dmma1688(acc[i][j], a[i], b[j]);
        };
        if (krem >= KC) {
#pragma unroll
          for (int kk = 0; kk < KC; kk += 8) kstep(kk);
        } else {
#pragma unroll 1
          for (int kk = 0; kk < krem; kk += 8) kstep(kk);
        }
      };
      if (cmask == 0xFFFFu) chunk(std::false_type{});
      else chunk(std::true_type{});
    }
  }
  if (skip) return;
  // the warp's computed blocks of P: the loads of a row group first (independent), then the subtraction and the stores
#pragma unroll
  for (int bi = 0; bi < 4; ++bi) {
    const int i = bi >> 1, h = bi & 1;  // product row i, C half h
    const int a = ta * 64 + wa + bi * 8 + lr;
    double pold[4][2];
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int bq = tb * 64 + wb + j * 8 + 2 * lc + e;
        pold[j][e] = (((cmask >> (4 * bi + j)) & 1u) && a < n && bq < n) ? P[a + (size_t)ld * bq] : 0.0;
      }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (!((cmask >> (4 * bi + j)) & 1u)) continue;  // a block below the diagonal: written by the mirror of its twin
      const int bq = tb * 64 + wb + j * 8 + 2 * lc;
      const double c0 = acc[i][j][2 * h], c1 = acc[i][j][2 * h + 1];
      const double v0 = pold[j][0] - c0, v1 = pold[j][1] - c1;
      if (a < n && bq < n) {
        P[a + (size_t)ld * bq] = v0;
        if (bq + 1 < n) P[a + (size_t)ld * (bq + 1)] = v1;
        if ((mmask >> (4 * bi + j)) & 1u) {  // lower counterpart: rows = b range (contiguous in P), column a
          double *dst = P + bq + (size_t)ld * a;
          if (bq + 1 < n) *reinterpret_cast<double2 *>(dst) = make_double2(v0, v1);
          else *dst = v0;
        }
      }
      // column n of Y is w = U^-T nu: (Y^T Y)(a, n) = (Y^T w)(a)  =>  x += Y^T w   (kalman.cpp:112)
      if (a < n) {
        if (bq == n) x[a] += c0;
        if (bq + 1 == n) x[a] += c1;
      }
    }
  }
}

// =============================================================================================
// kernel 4: upd_finish — normalise_state, symmetrise, counters
// =============================================================================================
__global__ void __launch_bounds__(UPD_THREADS) upd_finish_kernel(const Sl2Dev d, int stream_lo, int staged,
                                                                  int only_normalise) {
  pdl_prologue();
  const int s = stream_lo + blockIdx.x;
  const int tid = threadIdx.x;
  const int nf = d.nfeat[s];
  const int n = SL2_NXV + 3 * nf;
  const int ld = d.ld;
  double *__restrict__ P = d.P + (size_t)s * ld * ld;
  const double *__restrict__ x = d.x + (size_t)s * ld;
  const size_t fb = (size_t)s * d.Nmax;
  const int m = only_normalise ? 0 : d.upd_m[s];
  __shared__ int s_cull;
  // ---- normalise_state (monoslam.cpp:616-637): P <- J P J^T, J = diag(I3, dqnorm, I6, I) ---------
  if (m > 0 || only_normalise) {
    __shared__ double J4[16];
    if (tid == 0) {
      const rd q[4] = {rd(x[3]), rd(x[4]), rd(x[5]), rd(x[6])};
      const rd qq = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
      for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j)  // motion_model.cpp:371-380 (quirk Q2)
          J4[i * 4 + j] = (i == j) ? ((rd(1.0) - q[i] * q[i] / (qq * qq)) / qq).v
                                   : ((-q[i]) * q[j] / (qq * qq * qq)).v;
    }
    __syncthreads();
    // rows 3..6 of every column: P(3:7, j) = J4 * P(3:7, j)
    for (int j = tid; j < n; j += UPD_THREADS) {
      double v[4], o[4];
      for (int k = 0; k < 4; ++k) v[k] = P[(3 + k) + (size_t)ld * j];
      for (int i = 0; i < 4; ++i) {
        rd a(0.0);
        for (int k = 0; k < 4; ++k) a = a + rd(J4[i * 4 + k]) * rd(v[k]);
        o[i] = a.v;
      }
      for (int k = 0; k < 4; ++k) P[(3 + k) + (size_t)ld * j] = o[k];
    }
    __syncthreads();
    // columns 3..6: Pxx part gets (J Pxx) J^T; rows >= 13 are the mirror of the updated Pxy
    for (int i = tid; i < n; i += UPD_THREADS) {
      if (i < SL2_NXV) {
        double v[4], o[4];
        for (int k = 0; k < 4; ++k) v[k] = P[i + (size_t)ld * (3 + k)];
        for (int c = 0; c < 4; ++c) {
          rd a(0.0);
          for (int k = 0; k < 4; ++k) a = a + rd(v[k]) * rd(J4[c * 4 + k]);
          o[c] = a.v;
        }
        for (int k = 0; k < 4; ++k) P[i + (size_t)ld * (3 + k)] = o[k];
      } else {
        for (int k = 0; k < 4; ++k) P[i + (size_t)ld * (3 + k)] = P[(3 + k) + (size_t)ld * i];
      }
    }
    __syncthreads();
  }
  // ---- symmetrise (monoslam.cpp:143-150): only the Pxx block can be asymmetric here ---------
  {
    const int i = tid % 13, j = (tid / 13) % 13;
    const double a = P[i + (size_t)ld * j], b = P[j + (size_t)ld * i];
    const double v = (rd(a) * rd(0.5) + rd(b) * rd(0.5)).v;
    __syncthreads();
    if (tid < 169) P[i + (size_t)ld * j] = v;
    __syncthreads();
  }
  // ---- bookkeeping: attempt / success counters (monoslam.cpp:479-496) ------------------------
  if (!staged && !only_normalise) {
    if (tid == 0) s_cull = 0;  // number of features delete_bad_features would cull
    __syncthreads();
    for (int i = tid; i < nf; i += UPD_THREADS) {
      int att = d.attempted[fb + i], suc = d.successful[fb + i];
      if (d.sel_rank[fb + i] >= 0) {
        att += 1;
        if (d.found[fb + i] == 1) suc += 1;  // a match the consensus rejected (2) is an unsuccessful attempt
        d.attempted[fb + i] = att;
        d.successful[fb + i] = suc;
      }
      // monoslam.cpp:650-653; lets the cull kernel of the fused step return at once when idle
      if (att >= d.min_attempts && (double)suc / (double)att < d.match_fraction) atomicAdd(&s_cull, 1);
    }
    __syncthreads();
    if (tid == 0) d.ncull[s] = s_cull;
  }
}

// ---- host-side shapes ---------------------------------------------------------------------------
// The upd_solve instantiation that covers the measurement capacity (NP 16-row panels) and its shared memory.
struct SolveKernel {
  void (*kern)(Sl2Dev, int);
  int np;
  size_t smem;
};
template <int NP>
SolveKernel solve_kernel_np() {
  return {upd_solve_kernel<NP>, NP, SolveLayout<NP>::SMEM_DOUBLES * sizeof(double)};
}
inline SolveKernel solve_kernel(int kmax) {
  const int p = (2 * upd_keven(kmax) + 15) / 16;  // panels of S at capacity
  return p <= 4 ? solve_kernel_np<4>()
                : (p <= 7 ? solve_kernel_np<7>()
                          : (p <= 10 ? solve_kernel_np<10>() : (p <= 13 ? solve_kernel_np<13>() : solve_kernel_np<16>())));
}
inline void solve_shape(int Nmax, int &nslab, int &warps) {
  const int ngroups = (SL2_NXV + 3 * Nmax + 1 + 7) / 8;
  nslab = (ngroups + SOLVE_MAX_WARPS - 1) / SOLVE_MAX_WARPS;
  warps = (ngroups + nslab - 1) / nslab;
}
constexpr size_t SYRK_SMEM = (size_t)2 * 2 * 32 * UPD_YS * sizeof(double);  // upd_syrk_kernel<32, 2>

}  // namespace

size_t sl2_update_smem_bytes(const Sl2Dev &d) {  // upd_chol
  return chol_smem_doubles(d.kmax) * sizeof(double);
}

cudaError_t sl2_configure_update(const Sl2Dev &d) {
  const SolveKernel solve = solve_kernel(d.kmax);
  const struct {
    const void *kern;
    size_t smem;
  } opt_in[] = {
      {(const void *)upd_hp_kernel<7>, hp_layout(d.kmax, d.ld, 0).bytes},
      {(const void *)upd_hp_kernel<13>, hp_layout(d.kmax, d.ld, 0).bytes},
      {(const void *)upd_hp2_kernel<7>, hp_layout(d.kmax, d.ld, 7).bytes},
      {(const void *)upd_hp2_kernel<13>, hp_layout(d.kmax, d.ld, 13).bytes},
      {(const void *)upd_chol_kernel, sl2_update_smem_bytes(d)},
      {(const void *)solve.kern, solve.smem},
      {(const void *)upd_syrk_kernel<32, 2>, SYRK_SMEM},
  };
  for (const auto &k : opt_in) {
    const cudaError_t e = cudaFuncSetAttribute(k.kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k.smem);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

// ev6 (optional): 6 events recorded around the 5 kernels (hp, chol, solve, syrk, finish)
cudaError_t sl2_launch_update(const Sl2Dev &d, int stream_lo, int stream_cnt, int staged_m,
                              const int *st_feat, const double *st_Hxv, const double *st_Hy,
                              const double *st_R, const double *st_nu, int only_normalise,
                              Sl2Queue q, cudaEvent_t *ev6) {
  if (stream_cnt <= 0) return cudaSuccess;
  cudaError_t e;
  auto mark = [&](int i) { return ev6 ? cudaEventRecord(ev6[i], q.stream) : cudaSuccess; };
  if ((e = mark(0)) != cudaSuccess) return e;
  // row blocks of H P / S per stream: spread over CTAs unless the batch already fills the GPU with two streams per SM
  // (then one CTA per stream is fastest: every CTA rebuilds the measurement list and H tables)
  const int hp_all = (2 * upd_keven(d.kmax) + HP_ROWS - 1) / HP_ROWS;
  const int hp_blocks = stream_cnt >= 2 * d.nsm ? 1 : hp_all;
  const bool pdl = sl2_use_pdl(stream_cnt);
  if (!only_normalise) {
    const dim3 grid(hp_blocks, stream_cnt);
    // the software-pipelined form: one CTA per stream, one state column per thread
    const bool piped = hp_blocks == 1 && SL2_NXV + 3 * d.Nmax <= HP_THREADS;
    const int kd = staged_m >= 0 ? 13 : 7;
    auto *k13 = piped ? upd_hp2_kernel<13> : upd_hp_kernel<13>;
    auto *k7 = piped ? upd_hp2_kernel<7> : upd_hp_kernel<7>;
    const size_t smem = hp_layout(d.kmax, d.ld, piped ? kd : 0).bytes;
    e = sl2_launch_kernel(kd == 13 ? k13 : k7, grid, dim3(HP_THREADS), smem, q, pdl, d, stream_lo, staged_m,
                          st_feat, st_Hxv, st_Hy, st_R, st_nu);
    if (e != cudaSuccess) return e;
  }
  if ((e = mark(1)) != cudaSuccess) return e;
  if (!only_normalise) {
    e = sl2_launch_kernel(upd_chol_kernel, dim3(stream_cnt), dim3(UPD_THREADS), sl2_update_smem_bytes(d), q, pdl, d,
                          stream_lo);
    if (e != cudaSuccess) return e;
  }
  if ((e = mark(2)) != cudaSuccess) return e;
  if (!only_normalise) {
    int nslab, warps;
    solve_shape(d.Nmax, nslab, warps);
    const SolveKernel solve = solve_kernel(d.kmax);
    // two warps per 8-column group; a batch that fills the GPU runs one CTA per stream (U staged once per
    // stream, groups walked inside), a small one spreads a stream over nslab CTAs (latency)
    const bool walk = solve.np <= 13 && stream_cnt >= d.nsm;
    if (walk) warps = SOLVE_MAX_WARPS;
    e = sl2_launch_kernel(solve.kern, dim3(walk ? 1 : nslab, stream_cnt), dim3(64 * warps), solve.smem, q, pdl, d,
                          stream_lo);
    if (e != cudaSuccess) return e;
  }
  if ((e = mark(3)) != cudaSuccess) return e;
  if (!only_normalise) {
    // one 64x64 tile per CTA (CTAs that walk several tiles with cross-tile prefetch measured slower: they cost the
    // third resident CTA per SM)
    const int nt = (SL2_NXV + 3 * d.Nmax + 1 + 63) / 64;
    e = sl2_launch_kernel(upd_syrk_kernel<32, 2>, dim3(nt * (nt + 1) / 2, stream_cnt), dim3(SYRK_THREADS), SYRK_SMEM,
                          q, pdl, d, stream_lo);
    if (e != cudaSuccess) return e;
  }
  if ((e = mark(4)) != cudaSuccess) return e;
  e = sl2_launch_kernel(upd_finish_kernel, dim3(stream_cnt), dim3(UPD_THREADS), 0, q, pdl, d, stream_lo,
                        (int)(staged_m >= 0), only_normalise);
  if (e != cudaSuccess) return e;
  if ((e = mark(5)) != cudaSuccess) return e;
  return cudaGetLastError();
}
