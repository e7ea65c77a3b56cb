// snapshot.cu — stream snapshots: pack a batch of camera streams into blobs of the format of include/sl2b200.h,
// check the index fields of device blobs, and unpack blobs into streams.  One launch per batch, grid (blob, chunk).
// P dominates the bytes (0.78 MB per stream at n = 313, 4.9 MB at n = 781): it is copied one column per warp, and a
// column is contiguous on both sides (stride ld in the context, n in the blob), so every load and store of a warp
// covers 32 consecutive doubles.  The packed columns are only 16-byte aligned when n is even, hence 8-byte accesses.
// Entry points: sl2_snapshot_bytes / sl2_snapshot_layout, sl2_save_streams* and sl2_load_streams*, which check every
// blob's header on the host (snap_validate) and its index fields with the rule snap_index_ok states once for both.
#include <algorithm>

#include "sl2_context.cuh"

using namespace sl2;

// Section field[k] of a blob is the stream's first nfeat records of array k of SL2_STREAM_ARRAYS (x, P and the
// templates are laid out separately).
struct Sl2SnapLayout {
  size_t x, P, field[SL2_SNAPSHOT_FIELDS], templates, total;  // byte offsets in the blob, total size
};
__host__ __device__ inline size_t sl2_snap_align8(size_t b) { return (b + 7) & ~(size_t)7; }
__host__ __device__ inline Sl2SnapLayout sl2_snap_layout(int nfeat, int box) {
  Sl2SnapLayout L;
  const size_t n = SL2_NXV + 3 * (size_t)nfeat;
  size_t o = sizeof(sl2_snapshot_header);
  L.x = o;
  o += sl2_snap_align8(8 * n);
  L.P = o;
  o += 8 * n * n;
#define SL2_SECTION(T, name, per, by, reset) \
  L.field[SL2_FIELD_##name] = o;             \
  o += sl2_snap_align8((size_t)nfeat * per * sizeof(T));
  SL2_STREAM_ARRAYS(SL2_SECTION)
#undef SL2_SECTION
  L.templates = o;
  o += sl2_snap_align8((size_t)nfeat * box * box);
  L.total = o;
  return L;
}

// what the host validated for one blob of a load: the kernels take sizes and counts from here, never from the blob
struct Sl2SnapLoad {
  Sl2StreamCam cam;
  int stream, nfeat, nsel, nvisible, nmeas, ncull;
  int pad_[2];
};

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
    sl2_cam_config(d.cams[s], &u.h.cam);
    u.h.nsel = d.nsel[s];
    u.h.nvisible = d.nvisible[s];
    u.h.nmeas = d.nmeas[s];
    u.h.ncull = d.ncull[s];
    unsigned long long *hw = reinterpret_cast<unsigned long long *>(blob);
    for (int k = 0; k < 16; ++k) hw[k] = u.w[k];
  }
}

// The index rule of a load for feature f of a blob with nsel selected of nfeat features (include/sl2b200.h): its
// sel_rank r is -1 or a rank below both; its job_feat j names a feature or, below nsel, may be empty (-1), and is -1
// above nsel (the cull writes job slot sel_rank)
__host__ __device__ inline bool snap_index_ok(int f, int r, int j, int nsel, int nfeat) {
  return (r == -1 || (r >= 0 && r < nsel && r < nfeat)) && (f < nsel ? (j >= -1 && j < nfeat) : j == -1);
}

// the index rule for blob blockIdx.x, with the host-validated nfeat and nsel
__global__ void __launch_bounds__(SNAP_THREADS) snap_check_kernel(const Sl2Dev d, const Sl2SnapLoad *ld,
                                                                  const uint8_t *buf, size_t stride, int *bad) {
  const Sl2SnapLoad q = ld[blockIdx.x];
  const Sl2SnapLayout L = sl2_snap_layout(q.nfeat, d.box);
  const uint8_t *blob = buf + (size_t)blockIdx.x * stride;
  const int *rank = reinterpret_cast<const int *>(blob + L.field[SL2_FIELD_sel_rank]);
  const int *job = reinterpret_cast<const int *>(blob + L.field[SL2_FIELD_job_feat]);
  int ok = 1;
  for (int f = threadIdx.x; f < q.nfeat; f += blockDim.x) ok &= snap_index_ok(f, rank[f], job[f], q.nsel, q.nfeat);
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

// pack the streams [lo, lo + cnt) into blobs at buf + i * stride (nfeat read on the device, header written)
cudaError_t sl2_launch_pack(const Sl2Dev &d, int lo, int cnt, uint8_t *buf, size_t stride, Sl2Queue q) {
  if (cnt <= 0) return cudaSuccess;
  return sl2_launch_kernel(pack_streams_kernel, dim3(cnt, snap_chunks(d)), dim3(SNAP_THREADS), 0, q, false, d, lo, buf,
                           stride);
}

// adds the number of blobs whose job_feat / sel_rank fail the index rule (with the validated counts) to *bad
cudaError_t sl2_launch_snap_check(const Sl2Dev &d, int cnt, const Sl2SnapLoad *ld_dev, const uint8_t *buf,
                                  size_t stride, int *bad, Sl2Queue q) {
  if (cnt <= 0) return cudaSuccess;
  return sl2_launch_kernel(snap_check_kernel, dim3(cnt), dim3(SNAP_THREADS), 0, q, false, d, ld_dev, buf, stride, bad);
}

// unpack blob i into stream ld_dev[i].stream and reset what the blob does not cover
cudaError_t sl2_launch_unpack(const Sl2Dev &d, int cnt, const Sl2SnapLoad *ld_dev, const uint8_t *buf, size_t stride,
                              Sl2Queue q) {
  if (cnt <= 0) return cudaSuccess;
  return sl2_launch_kernel(unpack_streams_kernel, dim3(cnt, snap_chunks(d)), dim3(SNAP_THREADS), 0, q, false, d, ld_dev,
                           buf, stride);
}

// Checks the header of one blob (and, with `index`, its job_feat / sel_rank) against this context; fills `q` with
// the validated counts for stream s.  `blob` is host memory of at least `avail` bytes, any alignment.
int snap_validate(sl2_ctx *c, const uint8_t *blob, size_t stride, bool index, int s, Sl2SnapLoad *q,
                  const std::string &who) {
  sl2_snapshot_header h;
  memcpy(&h, blob, sizeof h);
  if (h.magic != SL2_SNAPSHOT_MAGIC || h.version != SL2_SNAPSHOT_VERSION || h.header_bytes != sizeof h)
    return fail(c, SL2_ERR_ARG, who + ": not a snapshot of this version and byte order");
  if (h.reserved0 != 0 || h.reserved1 != 0) return fail(c, SL2_ERR_ARG, who + ": reserved header fields are not 0");
  if (h.total_bytes > stride) return fail(c, SL2_ERR_ARG, who + ": blob larger than the stride");
  if (h.nfeat < 0 || h.nsel < 0 || h.nvisible < 0 || h.nmeas < 0 || h.ncull < 0)
    return fail(c, SL2_ERR_ARG, who + ": negative count");
  if ((int64_t)h.n != SL2_NXV + 3 * (int64_t)h.nfeat) return fail(c, SL2_ERR_ARG, who + ": n != 13 + 3 nfeat");
  if (h.boxsize != c->cfg.boxsize) return fail(c, SL2_ERR_ARG, who + ": boxsize differs from the context's");
  if (h.nfeat > c->cfg.max_features) return fail(c, SL2_ERR_STATE, who + ": map larger than max_features");
  const Sl2SnapLayout L = sl2_snap_layout(h.nfeat, h.boxsize);
  if (h.total_bytes != L.total) return fail(c, SL2_ERR_ARG, who + ": total size does not match nfeat and boxsize");
  // the counts are not renewed by a cull, sl2_delete_feature or sl2_set_features, so they are bounded by what any
  // prediction / update can produce, not by nfeat (include/sl2b200.h)
  if (h.nsel > SL2_MAX_MEASURED || h.nmeas > SL2_MAX_MEASURED || h.nvisible > SL2_MAX_FEATURES ||
      h.ncull > SL2_MAX_FEATURES)
    return fail(c, SL2_ERR_ARG, who + ": count above what a step can produce");
  const int rc = check_stream_config(c, &h.cam, who);
  if (rc) return rc;
  if (index) {
    for (int f = 0; f < h.nfeat; ++f) {
      int32_t r, j;
      memcpy(&r, blob + L.field[SL2_FIELD_sel_rank] + 4 * (size_t)f, 4);
      memcpy(&j, blob + L.field[SL2_FIELD_job_feat] + 4 * (size_t)f, 4);
      if (!snap_index_ok(f, r, j, h.nsel, h.nfeat))
        return fail(c, SL2_ERR_ARG, who + ": sel_rank or job_feat out of range");
    }
  }
  memset(q, 0, sizeof *q);
  q->cam = sl2_cam_row(h.cam);
  q->stream = s;
  q->nfeat = h.nfeat;
  q->nsel = h.nsel;
  q->nvisible = h.nvisible;
  q->nmeas = h.nmeas;
  q->ncull = h.ncull;
  return SL2_OK;
}

// The host forms stage groups of streams of at most this many bytes (at least one stream), so a save or load of a
// whole large context does not grow the staging buffers to the size of all its blobs.
const size_t SL2_SNAP_STAGE_BYTES = (size_t)64 << 20;
int snap_group(size_t sb) { return (int)std::max<size_t>(1, SL2_SNAP_STAGE_BYTES / sb); }

}  // namespace

extern "C" {

size_t sl2_snapshot_bytes(const sl2_ctx *c) { return c ? sl2_snap_layout(c->cfg.max_features, c->cfg.boxsize).total : 0; }

int sl2_snapshot_layout(int32_t nfeat, int32_t boxsize, sl2_snapshot_sections *out) {
  if (nfeat < 0 || nfeat > SL2_MAX_FEATURES || boxsize <= 0 || !out) return SL2_ERR_ARG;
  const Sl2SnapLayout L = sl2_snap_layout(nfeat, boxsize);
  out->x = L.x;
  out->P = L.P;
  for (int k = 0; k < SL2_SNAPSHOT_FIELDS; ++k) out->field[k] = L.field[k];
  out->templates = L.templates;
  out->total = L.total;
  return SL2_OK;
}

int sl2_save_streams(sl2_ctx *c, int32_t lo, int32_t cnt, void *buf, size_t stride, size_t *sizes) {
  if (bad_range(c, lo, cnt) || (cnt && !buf)) return fail(c, SL2_ERR_ARG, "sl2_save_streams: bad argument");
  const size_t sb = sl2_snapshot_bytes(c);
  if (stride < sb) return fail(c, SL2_ERR_ARG, "sl2_save_streams: stride below sl2_snapshot_bytes");
  if (cnt == 0) return SL2_OK;
  const int g = std::min(cnt, snap_group(sb));
  int rc = stage_reserve(c, (size_t)g * sb);
  if (rc) return rc;
  CU_TRY(c, cudaStreamSynchronize(c->stream));  // staging buffer reuse
  for (int i0 = 0; i0 < cnt; i0 += g) {
    const int k = std::min(g, cnt - i0);
    CU_TRY(c, sl2_launch_pack(c->d, lo + i0, k, c->stg_dev.get(), sb, queue(c)));
    CU_TRY(c, cudaMemcpyAsync(c->stg_host.get(), c->stg_dev.get(), (size_t)k * sb, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    for (int i = 0; i < k; ++i) {
      sl2_snapshot_header h;
      memcpy(&h, c->stg_host.get() + (size_t)i * sb, sizeof h);
      memcpy(static_cast<uint8_t *>(buf) + (size_t)(i0 + i) * stride, c->stg_host.get() + (size_t)i * sb, h.total_bytes);
      if (sizes) sizes[i0 + i] = h.total_bytes;
    }
  }
  return SL2_OK;
}

int sl2_save_streams_dev(sl2_ctx *c, int32_t lo, int32_t cnt, void *buf_dev, size_t stride) {
  if (bad_range(c, lo, cnt) || (cnt && !buf_dev) || ((uintptr_t)buf_dev & 7) || (stride & 7))
    return fail(c, SL2_ERR_ARG, "sl2_save_streams_dev: bad argument");
  if (stride < sl2_snapshot_bytes(c)) return fail(c, SL2_ERR_ARG, "sl2_save_streams_dev: stride below sl2_snapshot_bytes");
  if (cnt == 0) return SL2_OK;
  CU_TRY(c, sl2_launch_pack(c->d, lo, cnt, static_cast<uint8_t *>(buf_dev), stride, queue(c)));
  return SL2_OK;
}

int sl2_load_streams(sl2_ctx *c, int32_t lo, int32_t cnt, const void *buf, size_t stride) {
  if (bad_range(c, lo, cnt) || (cnt && !buf) || stride < sizeof(sl2_snapshot_header))
    return fail(c, SL2_ERR_ARG, "sl2_load_streams: bad argument");
  if (cnt == 0) return SL2_OK;
  const uint8_t *in = static_cast<const uint8_t *>(buf);
  std::vector<Sl2SnapLoad> q(cnt);
  std::vector<sl2_stream_config> cams(cnt);
  for (int i = 0; i < cnt; ++i) {
    const int rc = snap_validate(c, in + (size_t)i * stride, stride, true, lo + i, &q[i], "sl2_load_streams");
    if (rc) return rc;
    memcpy(&cams[i], in + (size_t)i * stride + offsetof(sl2_snapshot_header, cam), sizeof(sl2_stream_config));
  }
  // staging, one group of streams at a time: its load records, then its blobs at the context's snapshot size
  const size_t sb = sl2_snapshot_bytes(c);
  const int g = std::min(cnt, snap_group(sb));
  const size_t pb = ((size_t)g * sizeof(Sl2SnapLoad) + 255) & ~(size_t)255;
  int rc = stage_reserve(c, pb + (size_t)g * sb);
  if (rc) return rc;
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  for (int i0 = 0; i0 < cnt; i0 += g) {
    const int k = std::min(g, cnt - i0);
    CU_TRY(c, cudaStreamSynchronize(c->stream));  // the previous group's unpack has read the staging buffer
    memcpy(c->stg_host.get(), q.data() + i0, (size_t)k * sizeof(Sl2SnapLoad));
    size_t end = 0;
    for (int i = 0; i < k; ++i) {
      const size_t tb = sl2_snap_layout(q[i0 + i].nfeat, c->cfg.boxsize).total;
      memcpy(c->stg_host.get() + pb + (size_t)i * sb, in + (size_t)(i0 + i) * stride, tb);
      end = pb + (size_t)i * sb + tb;
    }
    CU_TRY(c, cudaMemcpyAsync(c->stg_dev.get(), c->stg_host.get(), end, cudaMemcpyHostToDevice, c->stream));
    CU_TRY(c, sl2_launch_unpack(c->d, k, reinterpret_cast<const Sl2SnapLoad *>(c->stg_dev.get()),
                                c->stg_dev.get() + pb, sb, queue(c)));
  }
  const int rf = streams_restarted(c, lo, cnt);
  if (rf) return rf;
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return loaded_cameras(c, lo, cams);
}

int sl2_load_streams_dev(sl2_ctx *c, int32_t lo, int32_t cnt, const void *buf_dev, size_t stride) {
  if (bad_range(c, lo, cnt) || (cnt && !buf_dev) || ((uintptr_t)buf_dev & 7) || (stride & 7) ||
      stride < sizeof(sl2_snapshot_header))
    return fail(c, SL2_ERR_ARG, "sl2_load_streams_dev: bad argument");
  if (cnt == 0) return SL2_OK;
  const uint8_t *in = static_cast<const uint8_t *>(buf_dev);
  const size_t hb = sizeof(sl2_snapshot_header);
  // staging: load records | verdict (int) | headers copied down
  const size_t pb = ((size_t)cnt * sizeof(Sl2SnapLoad) + 255) & ~(size_t)255, o_bad = pb, o_h = pb + 256;
  int rc = stage_reserve(c, o_h + (size_t)cnt * hb);
  if (rc) return rc;
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  CU_TRY(c, cudaMemcpy2DAsync(c->stg_host.get() + o_h, hb, in, stride, hb, cnt, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  std::vector<Sl2SnapLoad> q(cnt);
  std::vector<sl2_stream_config> cams(cnt);
  for (int i = 0; i < cnt; ++i) {
    const uint8_t *h = c->stg_host.get() + o_h + (size_t)i * hb;
    rc = snap_validate(c, h, stride, false, lo + i, &q[i], "sl2_load_streams_dev");
    if (rc) return rc;
    memcpy(&cams[i], h + offsetof(sl2_snapshot_header, cam), sizeof(sl2_stream_config));
  }
  memcpy(c->stg_host.get(), q.data(), (size_t)cnt * sizeof(Sl2SnapLoad));
  memset(c->stg_host.get() + o_bad, 0, sizeof(int));
  CU_TRY(c, cudaMemcpyAsync(c->stg_dev.get(), c->stg_host.get(), o_bad + sizeof(int), cudaMemcpyHostToDevice, c->stream));
  const Sl2SnapLoad *q_dev = reinterpret_cast<const Sl2SnapLoad *>(c->stg_dev.get());
  int *bad_dev = reinterpret_cast<int *>(c->stg_dev.get() + o_bad);
  CU_TRY(c, sl2_launch_snap_check(c->d, cnt, q_dev, in, stride, bad_dev, queue(c)));
  int bad = 0;
  CU_TRY(c, cudaMemcpyAsync(&bad, bad_dev, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  if (bad) return fail(c, SL2_ERR_ARG, "sl2_load_streams_dev: sel_rank or job_feat out of range");
  CU_TRY(c, sl2_launch_unpack(c->d, cnt, q_dev, in, stride, queue(c)));
  const int rf = streams_restarted(c, lo, cnt);
  if (rf) return rf;
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return loaded_cameras(c, lo, cams);
}

}  // extern "C"
