// snapshot.cu — stream snapshots: pack a batch of camera streams into blobs of the format of include/sl2b200.h,
// check the index fields of device blobs, and unpack blobs into streams.  One launch per batch, grid (blob, chunk).
// P dominates the bytes (0.78 MB per stream at n = 313, 4.9 MB at n = 781): it is copied one column per warp, and a
// column is contiguous on both sides (stride ld in the context, n in the blob), so every load and store of a warp
// covers 32 consecutive doubles.  The packed columns are only 16-byte aligned when n is even, hence 8-byte accesses.
#include "sl2_common.cuh"

namespace {

constexpr int SNAP_THREADS = 256;
constexpr int SNAP_WARPS = SNAP_THREADS / 32;
static_assert(sizeof(sl2_snapshot_header) == 128, "the header is 16 words");
static_assert(sizeof(Sl2SnapLoad) % 8 == 0, "load records are copied as one array");

// dst[r] = src[r] for r < cnt by one warp, four independent loads in flight per lane before their stores
__device__ __forceinline__ void warp_copy(const double *__restrict__ src, double *__restrict__ dst, int cnt,
                                          int lane) {
  int r = lane;
  for (; r + 96 < cnt; r += 128) {
    const double a = src[r], b = src[r + 32], c = src[r + 64], e = src[r + 96];
    dst[r] = a;
    dst[r + 32] = b;
    dst[r + 64] = c;
    dst[r + 96] = e;
  }
  for (; r < cnt; r += 32) dst[r] = src[r];
}

// dst[e] = e < cnt ? src[e] : fill for e < len, elements of type T, over the threads [t, T) of a stream
template <typename T>
__device__ __forceinline__ void copy_fill(const T *__restrict__ src, T *__restrict__ dst, size_t cnt, size_t len,
                                          T fill, size_t t, size_t nt) {
  for (size_t e = t; e < len; e += nt) dst[e] = e < cnt ? src[e] : fill;
}

__global__ void __launch_bounds__(SNAP_THREADS) pack_streams_kernel(const Sl2Dev d, int lo, uint8_t *buf,
                                                                    size_t stride) {
  const int i = blockIdx.x, s = lo + i, tid = threadIdx.x, lane = tid & 31;
  const int nf = d.nfeat[s], n = SL2_NXV + 3 * nf, ld = d.ld;
  const Sl2SnapLayout L = sl2_snap_layout(nf, d.box);
  uint8_t *blob = buf + (size_t)i * stride;
  // P: one warp per column
  const double *P = d.P + (size_t)s * ld * ld;
  double *Po = reinterpret_cast<double *>(blob + L.P);
  for (int c = blockIdx.y * SNAP_WARPS + (tid >> 5); c < n; c += gridDim.y * SNAP_WARPS)
    warp_copy(P + (size_t)ld * c, Po + (size_t)n * c, n, lane);
  // everything else over the threads of the stream's blocks; alignment padding is written as zeros
  const size_t t = (size_t)blockIdx.y * SNAP_THREADS + tid, nt = (size_t)gridDim.y * SNAP_THREADS;
  copy_fill(d.x + (size_t)s * ld, reinterpret_cast<double *>(blob + L.x), (size_t)n, (size_t)n, 0.0, t, nt);
  const size_t fb = (size_t)s * d.Nmax;
#define SL2_PACK(T, name, per, by, reset)                                                                       \
  copy_fill(d.name + fb * per, reinterpret_cast<T *>(blob + L.field[SL2_FIELD_##name]), (size_t)nf * per,       \
            sl2_snap_align8((size_t)nf * per * sizeof(T)) / sizeof(T), (T)0, t, nt);
  SL2_STREAM_ARRAYS(SL2_PACK)
#undef SL2_PACK
  // templates: rows of box bytes out of the device's 16-byte rows
  const int box = d.box, bb = box * box;
  const uint8_t *pt = d.patches + fb * box * 16;
  const size_t tb = (size_t)nf * bb;
  for (size_t e = t; e < sl2_snap_align8(tb); e += nt) {
    uint8_t v = 0;
    if (e < tb) {
      const int f = (int)(e / bb), rem = (int)(e - (size_t)f * bb), r = rem / box;
      v = pt[((size_t)f * box + r) * 16 + (rem - r * box)];
    }
    blob[L.templates + e] = v;
  }
  if (blockIdx.y == 0 && tid == 0) {
    union {
      sl2_snapshot_header h;
      unsigned long long w[16];
    } u;
    for (int k = 0; k < 16; ++k) u.w[k] = 0ull;  // padding bytes included: the blob is canonical
    u.h.magic = SL2_SNAPSHOT_MAGIC;
    u.h.version = SL2_SNAPSHOT_VERSION;
    u.h.header_bytes = sizeof(sl2_snapshot_header);
    u.h.total_bytes = L.total;
    u.h.boxsize = box;
    u.h.nfeat = nf;
    u.h.n = n;
    const Sl2StreamCam &cr = d.cams[s];
    u.h.cam.width = (int32_t)cr.cam[0];
    u.h.cam.height = (int32_t)cr.cam[1];
    u.h.cam.fku = cr.cam[2];
    u.h.cam.fkv = cr.cam[3];
    u.h.cam.u0 = cr.cam[4];
    u.h.cam.v0 = cr.cam[5];
    u.h.cam.kd1 = cr.cam[6];
    u.h.cam.sd = cr.cam[7];
    u.h.cam.delta_t = cr.dt;
    u.h.cam.number_of_features_to_select = cr.n_select;
    u.h.nsel = d.nsel[s];
    u.h.nvisible = d.nvisible[s];
    u.h.nmeas = d.nmeas[s];
    u.h.ncull = d.ncull[s];
    unsigned long long *hw = reinterpret_cast<unsigned long long *>(blob);
    for (int k = 0; k < 16; ++k) hw[k] = u.w[k];
  }
}

// the index rules of a load for blob blockIdx.x, with the host-validated nfeat and nsel (include/sl2b200.h)
__global__ void __launch_bounds__(SNAP_THREADS) snap_check_kernel(const Sl2Dev d, const Sl2SnapLoad *ld,
                                                                  const uint8_t *buf, size_t stride, int *bad) {
  const Sl2SnapLoad q = ld[blockIdx.x];
  const Sl2SnapLayout L = sl2_snap_layout(q.nfeat, d.box);
  const uint8_t *blob = buf + (size_t)blockIdx.x * stride;
  const int *rank = reinterpret_cast<const int *>(blob + L.field[SL2_FIELD_sel_rank]);
  const int *job = reinterpret_cast<const int *>(blob + L.field[SL2_FIELD_job_feat]);
  int ok = 1;
  for (int f = threadIdx.x; f < q.nfeat; f += blockDim.x) {
    const int r = rank[f], j = job[f];
    ok &= (r == -1 || (r >= 0 && r < q.nsel && r < q.nfeat));
    ok &= f < q.nsel ? (j >= -1 && j < q.nfeat) : (j == -1);
  }
  if (!__syncthreads_and(ok) && threadIdx.x == 0) atomicAdd(bad, 1);
}

__global__ void __launch_bounds__(SNAP_THREADS) unpack_streams_kernel(const Sl2Dev d, const Sl2SnapLoad *ldv,
                                                                      const uint8_t *buf, size_t stride) {
  const int i = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
  const Sl2SnapLoad &q = ldv[i];  // read where used: the camera row only by the thread that writes it
  const int s = q.stream, nf = q.nfeat, n = SL2_NXV + 3 * nf, ld = d.ld;
  const Sl2SnapLayout L = sl2_snap_layout(nf, d.box);
  const uint8_t *blob = buf + (size_t)i * stride;
  // P: one warp per column of the whole ld x ld block, zero outside n x n
  double *P = d.P + (size_t)s * ld * ld;
  const double *Pi = reinterpret_cast<const double *>(blob + L.P);
  for (int c = blockIdx.y * SNAP_WARPS + (tid >> 5); c < ld; c += gridDim.y * SNAP_WARPS) {
    double *col = P + (size_t)ld * c;
    const int rows = c < n ? n : 0;
    if (rows) warp_copy(Pi + (size_t)n * c, col, rows, lane);
    for (int r = rows + lane; r < ld; r += 32) col[r] = 0.0;
  }
  const size_t t = (size_t)blockIdx.y * SNAP_THREADS + tid, nt = (size_t)gridDim.y * SNAP_THREADS;
  copy_fill(reinterpret_cast<const double *>(blob + L.x), d.x + (size_t)s * ld, (size_t)n, (size_t)ld, 0.0, t, nt);
  const size_t fb = (size_t)s * d.Nmax;
#define SL2_UNPACK(T, name, per, by, reset)                                                                     \
  copy_fill(reinterpret_cast<const T *>(blob + L.field[SL2_FIELD_##name]), d.name + fb * per, (size_t)nf * per, \
            (size_t)d.Nmax * per, (T)(reset), t, nt);
  SL2_STREAM_ARRAYS(SL2_UNPACK)
#undef SL2_UNPACK
  const int box = d.box, b16 = box * 16;
  uint8_t *pt = d.patches + fb * b16;
  const uint8_t *tp = blob + L.templates;
  for (size_t e = t; e < (size_t)d.Nmax * b16; e += nt) {
    const int f = (int)(e / b16), rem = (int)(e - (size_t)f * b16), r = rem >> 4, col = rem & 15;
    pt[e] = (f < nf && col < box) ? tp[((size_t)f * box + r) * box + col] : (uint8_t)0;
  }
  if (blockIdx.y == 0 && tid == 0) {
    d.nfeat[s] = nf;
    d.nsel[s] = q.nsel;
    d.nvisible[s] = q.nvisible;
    d.nmeas[s] = q.nmeas;
    d.ncull[s] = q.ncull;
    d.cams[s] = q.cam;
  }
}

// blocks per stream: about two columns of P per warp at the context's capacity
int snap_chunks(const Sl2Dev &d) { return (d.ld + 2 * SNAP_WARPS - 1) / (2 * SNAP_WARPS); }

}  // namespace

cudaError_t sl2_launch_pack(const Sl2Dev &d, int lo, int cnt, uint8_t *buf, size_t stride, Sl2Queue q) {
  if (cnt <= 0) return cudaSuccess;
  return sl2_launch_kernel(pack_streams_kernel, dim3(cnt, snap_chunks(d)), dim3(SNAP_THREADS), 0, q, false, d, lo, buf,
                           stride);
}

cudaError_t sl2_launch_snap_check(const Sl2Dev &d, int cnt, const Sl2SnapLoad *ld_dev, const uint8_t *buf,
                                  size_t stride, int *bad, Sl2Queue q) {
  if (cnt <= 0) return cudaSuccess;
  return sl2_launch_kernel(snap_check_kernel, dim3(cnt), dim3(SNAP_THREADS), 0, q, false, d, ld_dev, buf, stride, bad);
}

cudaError_t sl2_launch_unpack(const Sl2Dev &d, int cnt, const Sl2SnapLoad *ld_dev, const uint8_t *buf, size_t stride,
                              Sl2Queue q) {
  if (cnt <= 0) return cudaSuccess;
  return sl2_launch_kernel(unpack_streams_kernel, dim3(cnt, snap_chunks(d)), dim3(SNAP_THREADS), 0, q, false, d, ld_dev,
                           buf, stride);
}
