// ingest.cu — raw camera frames to the gray frame ring: the cvtColor + resize of the reference's camera grabber
// (framegrabber/usbcamgrabber.cpp:75-113) on the device, for every stream with a source (sl2_set_stream_source).
//
// Arithmetic (bit-exact, integer except the resize coordinates):
//   RGB24 -> gray   OpenCV 2.4 RGB2Gray<uchar> (color.cpp: yuv_shift = 14, R2Y = 4899, G2Y = 9617, B2Y = 1868):
//                   (4899 R + 9617 G + 1868 B + 8192) >> 14.  The reference pins OpenCV 2.4.2; OpenCV 4 computes
//                   (9798 R + 19235 G + 3735 B + 16384) >> 15, which differs on some colours by one grey level.
//   UYVY -> gray    byte 1 of every 2-byte pixel (CV_YUV2GRAY_Y422 == CV_YUV2GRAY_UYVY).  A YUYV camera would feed
//                   chroma as gray, as in the reference.
//   GRAY8           the byte.
//   resize          OpenCV's 8-bit INTER_LINEAR of the rounded gray image, to the stream's image size:
//                   - same size: a copy; exactly 2x in both directions: (a + b + c + d + 2) >> 2 (OpenCV turns this
//                     case into INTER_AREA's fast path in every version);
//                   - otherwise, per axis with scale = 1 / (dst / src) in double: f = float((d + 0.5) scale - 0.5),
//                     i = floor(f), f -= i, weights rint((1 - f) 2048), rint(f 2048).  Columns clamp at both borders
//                     (i < 0 -> i = 0, f = 0; i >= src - 1 -> i = src - 1, f = 0); rows keep their weights and clamp
//                     the row index.  Horizontal sums S = g0 a0 + g1 a1, vertical
//                     (((b0 (S0 >> 4)) >> 16) + ((b1 (S1 >> 4)) >> 16) + 2) >> 2 (the SIMD path of
//                     VResizeLinearVec_32s8u).
//                   Pinned to OpenCV 4.13's cv2.resize (tests/ingest_ref.py); OpenCV 2.4.2's resize cannot be run
//                   beside it, so only the 2x case is shown version-independent.
//
// One launch covers the streams of a frame copy: block (band, row) converts output rows [band * ROWS, ...) of table
// row base + blockIdx.y.  The raw source rows an output row needs are loaded once into shared memory with aligned
// 16-byte loads and converted there (gray is recomputed per use, which is exact); consecutive output rows reuse them.
//
// Host side: sl2_set_stream_source builds the table of streams with a source and their raw frames' staging
// (install_sources); sl2_set_frame / sl2_set_frames* and the asynchronous step copy a frame set into the ring or the
// staging (copy_slot_frames), then convert.
#include <algorithm>

#include "sl2_context.cuh"

using namespace sl2;

#define SL2_SOURCE_CHUNK 64  // rows one table write carries as its kernel parameter
struct Sl2SourceChunk {
  int first, n;
  Sl2Source row[SL2_SOURCE_CHUNK];
};

namespace {

constexpr int INGEST_THREADS = 256;
constexpr int INGEST_ROWS = 4;  // output rows per block

__global__ void source_write_kernel(Sl2Source *table, const Sl2SourceChunk chunk) {
  const int i = threadIdx.x;
  if (i < chunk.n) table[chunk.first + i] = chunk.row[i];
}

__device__ __forceinline__ int gray_at(const uint8_t *row, int x, int format) {
  if (format == SL2_SRC_RGB24) {
    const uint8_t *p = row + 3 * x;
    return (4899 * p[0] + 9617 * p[1] + 1868 * p[2] + 8192) >> 14;
  }
  if (format == SL2_SRC_UYVY) return row[2 * x + 1];
  return row[x];
}

// OpenCV's INTER_LINEAR source coordinate of destination index d: index and 11-bit weights (w0, w1)
struct Tap {
  int i, w0, w1;
};
__device__ __forceinline__ Tap linear_tap(int d, double scale, int src, bool clamp) {
  const float f = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn((double)d, 0.5), scale), 0.5));
  const float fl = floorf(f);
  int i = (int)fl;
  float fr = __fsub_rn(f, fl);
  if (clamp) {
    if (i < 0) i = 0, fr = 0.f;
    if (i >= src - 1) i = src - 1, fr = 0.f;
  }
  return {i, __float2int_rn(__fmul_rn(__fsub_rn(1.f, fr), 2048.f)), __float2int_rn(__fmul_rn(fr, 2048.f))};
}

__device__ __forceinline__ int shift_of(const uint8_t *p) { return (int)((uintptr_t)p & 15); }

// bytes [src, src + n) of global memory -> smem (16-byte aligned) from smem + shift_of(src) on, by 16-byte loads of
// the aligned words covering them.  The staging area is 16-byte aligned per slot with 16 bytes of slack at its end.
__device__ __forceinline__ void load_row(uint8_t *smem, const uint8_t *src, int n) {
  const int words = (shift_of(src) + n + 15) >> 4;
  const uint4 *g = reinterpret_cast<const uint4 *>(src - shift_of(src));
  uint4 *s = reinterpret_cast<uint4 *>(smem);
  for (int w = threadIdx.x; w < words; w += blockDim.x) s[w] = __ldg(g + w);
}

__global__ void __launch_bounds__(INGEST_THREADS) ingest_kernel(const Sl2Source *table, int base,
                                                                const uint8_t *stage, uint8_t *ring_slot, int H,
                                                                int pitch, int row_cap) {
  extern __shared__ __align__(16) uint8_t sm[];
  const Sl2Source src = table[base + blockIdx.y];
  const int y0 = blockIdx.x * INGEST_ROWS;
  if (y0 >= src.dh) return;
  const int y1 = min(y0 + INGEST_ROWS, src.dh);
  const int bpp = src.format == SL2_SRC_RGB24 ? 3 : src.format == SL2_SRC_UYVY ? 2 : 1;
  const int rb = src.sw * bpp;
  const uint8_t *raw = stage + src.off;
  uint8_t *out = ring_slot + (size_t)src.stream * H * pitch;
  const bool same = src.sw == src.dw && src.sh == src.dh;
  const bool half = src.sw == 2 * src.dw && src.sh == 2 * src.dh;
  const double sx = 1.0 / ((double)src.dw / src.sw), sy = 1.0 / ((double)src.dh / src.sh);
  int h0 = -1, h1 = -1, b0k = 0, b1k = 1;  // source row held by, and index of, the buffer of r0 / r1
  for (int y = y0; y < y1; ++y) {
    int r0, r1, b0 = 2048, b1 = 0;
    if (same) {
      r0 = r1 = y;
    } else if (half) {
      r0 = 2 * y, r1 = 2 * y + 1;
    } else {
      const Tap t = linear_tap(y, sy, src.sh, false);
      r0 = min(max(t.i, 0), src.sh - 1);
      r1 = min(max(t.i + 1, 0), src.sh - 1);
      b0 = t.w0, b1 = t.w1;
    }
    // buffer k (at sm + bk * row_cap) must hold row rk; a held row that is still needed stays where it is
    if (h1 == r0 || h0 == r1) {
      const int tb = b0k, th = h0;
      b0k = b1k, h0 = h1;
      b1k = tb, h1 = th;
    }
    __syncthreads();  // every thread is done with the rows about to be replaced
    if (h0 != r0) load_row(sm + b0k * row_cap, raw + (size_t)r0 * rb, rb), h0 = r0;
    if (!same && h1 != r1) load_row(sm + b1k * row_cap, raw + (size_t)r1 * rb, rb), h1 = r1;
    __syncthreads();
    uint8_t *o = out + (size_t)y * pitch;
    const uint8_t *g0 = sm + b0k * row_cap + shift_of(raw + (size_t)r0 * rb);
    const uint8_t *g1 = sm + b1k * row_cap + shift_of(raw + (size_t)r1 * rb);
    for (int x = threadIdx.x; x < src.dw; x += blockDim.x) {
      int v;
      if (same) {
        v = gray_at(g0, x, src.format);
      } else if (half) {
        v = (gray_at(g0, 2 * x, src.format) + gray_at(g0, 2 * x + 1, src.format) + gray_at(g1, 2 * x, src.format) +
             gray_at(g1, 2 * x + 1, src.format) + 2) >> 2;
      } else {
        const Tap t = linear_tap(x, sx, src.sw, true);
        const int x1 = min(t.i + 1, src.sw - 1);
        const int s0 = gray_at(g0, t.i, src.format) * t.w0 + gray_at(g0, x1, src.format) * t.w1;
        const int s1 = gray_at(g1, t.i, src.format) * t.w0 + gray_at(g1, x1, src.format) * t.w1;
        v = (((b0 * (s0 >> 4)) >> 16) + ((b1 * (s1 >> 4)) >> 16) + 2) >> 2;
      }
      o[x] = (uint8_t)v;
    }
  }
}

int sl2_source_bpp(int format) { return format == SL2_SRC_RGB24 ? 3 : format == SL2_SRC_UYVY ? 2 : 1; }

// table[first .. first + n) = the chunk's rows, ordered on the queue like any other launch
cudaError_t sl2_launch_source_write(Sl2Source *table, const Sl2SourceChunk &chunk, Sl2Queue q) {
  return sl2_launch_kernel(source_write_kernel, dim3(1), dim3(SL2_SOURCE_CHUNK), 0, q, false, table, chunk);
}

// convert (and resize) the raw frames of table rows [base, base + cnt) from one slot of the staging area into the
// ring slot `slot`; max_row_bytes = the largest sw * bpp of those rows
cudaError_t sl2_launch_ingest(const Sl2Dev &d, const Sl2Source *table, int base, int cnt, int max_dh,
                              int max_row_bytes, const uint8_t *stage_slot, int slot, Sl2Queue q) {
  if (cnt <= 0) return cudaSuccess;
  const int row_cap = ((max_row_bytes + 15) & ~15) + 16;  // one raw row at any 16-byte misalignment
  const dim3 grid((max_dh + INGEST_ROWS - 1) / INGEST_ROWS, cnt);
  uint8_t *ring_slot = d.frames + (size_t)slot * d.B * d.H * d.pitch;
  return sl2_launch_kernel(ingest_kernel, grid, dim3(INGEST_THREADS), 2 * (size_t)row_cap, q, false, table, base,
                           stage_slot, ring_slot, d.H, d.pitch, row_cap);
}

// gray blocks of the streams [lo, hi), [hi - lo][H][W] packed, into the frame ring
cudaError_t copy_gray_blocks(const Sl2Dev &d, int slot, int lo, int hi, const uint8_t *src, cudaMemcpyKind kind,
                             cudaStream_t st) {
  uint8_t *dst = d.frames + ((size_t)slot * d.B + lo) * d.H * d.pitch;
  if (d.pitch == d.W) return cudaMemcpyAsync(dst, src, (size_t)(hi - lo) * d.H * d.W, kind, st);
  return cudaMemcpy2DAsync(dst, d.pitch, src, d.W, d.W, (size_t)(hi - lo) * d.H, kind, st);
}

uint8_t *source_stage(const sl2_ctx *c, int slot) { return c->src_stage.get() + (size_t)slot * c->src_slot_bytes; }

// convert the raw frames of source rows [base, base + cnt) of `slot`'s staging into the ring
cudaError_t ingest(sl2_ctx *c, int slot, int base, int cnt, Sl2Queue q) {
  int max_dh = 0, max_rb = 0;
  for (int j = base; j < base + cnt; ++j) {
    const Sl2Source &r = c->src_rows[j];
    max_dh = std::max(max_dh, r.dh);
    max_rb = std::max(max_rb, r.sw * sl2_source_bpp(r.format));
  }
  return sl2_launch_ingest(c->d, c->src_tab.get(), base, cnt, max_dh, max_rb, source_stage(c, slot), slot, q);
}

size_t frame_bytes(const sl2_ctx *c, const sl2_stream_source &s) {
  return s.format == SL2_SRC_GRAY_RING ? (size_t)c->d.H * c->d.W
                                       : (size_t)s.width * s.height * sl2_source_bpp(s.format);
}

}  // namespace

namespace sl2 {

// Make `srcs` the context's sources (with the cameras in c->cams): layout, table rows, staging and the device table.
// The table is rewritten on `stream` after every conversion queued so far on the copy stream.
int install_sources(sl2_ctx *c, const std::vector<sl2_stream_source> &srcs) {
  const Sl2Dev &d = c->d;
  std::vector<size_t> layout(d.B + 1, 0);
  std::vector<Sl2Source> rows;
  size_t raw = 0;
  for (int s = 0; s < d.B; ++s) {
    layout[s + 1] = layout[s] + frame_bytes(c, srcs[s]);
    if (srcs[s].format == SL2_SRC_GRAY_RING) continue;
    rows.push_back({s, srcs[s].format, srcs[s].width, srcs[s].height, c->cams[s].width, c->cams[s].height,
                    (int64_t)raw});
    raw += frame_bytes(c, srcs[s]);
  }
  const size_t slot_bytes = (raw + 15) & ~(size_t)15;
  const size_t need = rows.empty() ? 0 : (size_t)d.slots * slot_bytes + 16;
  // every allocation before anything changes: a failed one leaves the sources, the staging and the table as they were
  DevPtr<uint8_t> stage;
  if (need > c->src_stage_bytes) {  // nothing may still read or write the old staging
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    CU_TRY(c, cudaStreamSynchronize(c->copy_stream.get()));
    CU_TRY(c, cuda_malloc(stage, need));
  }
  if (!rows.empty() && !c->src_tab) CU_TRY(c, cuda_malloc(c->src_tab, sizeof(Sl2Source) * d.B));
  if (!rows.empty() && !c->ev_src) CU_TRY(c, cuda_event_create(c->ev_src, cudaEventDisableTiming));
  if (stage) {
    c->src_stage = std::move(stage);
    c->src_stage_bytes = need;
  }
  if (!rows.empty()) {
    for (const SlotEvents &e : c->ev_slot)  // conversions in flight
      CU_TRY(c, cudaStreamWaitEvent(c->stream, e.h2d.get(), 0));
    for (size_t first = 0; first < rows.size(); first += SL2_SOURCE_CHUNK) {
      Sl2SourceChunk ch = {};
      ch.first = (int)first;
      ch.n = (int)std::min(rows.size() - first, (size_t)SL2_SOURCE_CHUNK);
      for (int i = 0; i < ch.n; ++i) ch.row[i] = rows[first + i];
      CU_TRY(c, sl2_launch_source_write(c->src_tab.get(), ch, queue(c)));
    }
    CU_TRY(c, cudaEventRecord(c->ev_src.get(), c->stream));
  }
  c->srcs = srcs;
  c->layout = layout;
  c->src_rows = rows;
  c->src_slot_bytes = slot_bytes;
  return SL2_OK;
}

// A snapshot load gives streams [lo, lo + cnt) the blobs' cameras: a stream with a source then resizes to its new image
int loaded_cameras(sl2_ctx *c, int lo, const std::vector<sl2_stream_config> &cams) {
  bool resized = false;
  for (size_t i = 0; i < cams.size(); ++i) {
    const sl2_stream_config &old = c->cams[lo + i];
    resized = resized || (c->srcs[lo + i].format != SL2_SRC_GRAY_RING &&
                          (old.width != cams[i].width || old.height != cams[i].height));
    c->cams[lo + i] = cams[i];
  }
  return resized ? install_sources(c, c->srcs) : SL2_OK;
}

// One frame slot of every stream, a frame set (sl2_frame_set_layout), into the frame ring: each run of consecutive
// default streams in one copy to the ring (the whole set when no stream has a source), each run of streams with a
// source in one copy to the slot's staging, then one conversion launch for all of them.
cudaError_t copy_slot_frames(sl2_ctx *c, int slot, const uint8_t *src, cudaMemcpyKind kind, Sl2Queue q) {
  const Sl2Dev &d = c->d;
  if (c->src_rows.empty()) return copy_gray_blocks(d, slot, 0, d.B, src, kind, q.stream);
  for (int a = 0; a < d.B;) {
    const bool raw = c->srcs[a].format != SL2_SRC_GRAY_RING;
    int b = a + 1;
    while (b < d.B && (c->srcs[b].format != SL2_SRC_GRAY_RING) == raw) ++b;
    cudaError_t e;
    if (raw) {
      size_t at = 0;  // staging offset of stream a
      for (const Sl2Source &r : c->src_rows)
        if (r.stream == a) at = (size_t)r.off;
      e = cudaMemcpyAsync(source_stage(c, slot) + at, src + c->layout[a], c->layout[b] - c->layout[a], kind,
                          q.stream);
    } else {
      e = copy_gray_blocks(d, slot, a, b, src + c->layout[a], kind, q.stream);
    }
    if (e != cudaSuccess) return e;
    a = b;
  }
  return ingest(c, slot, 0, (int)c->src_rows.size(), q);
}

}  // namespace sl2

extern "C" {

int sl2_set_stream_source(sl2_ctx *c, int32_t s, const sl2_stream_source *src) {
  if (bad_stream(c, s) || !src) return fail(c, SL2_ERR_ARG, "sl2_set_stream_source: bad argument");
  const int f = src->format;
  if (f < SL2_SRC_GRAY_RING || f > SL2_SRC_UYVY || src->reserved != 0)
    return fail(c, SL2_ERR_ARG, "sl2_set_stream_source: unknown format or non-zero reserved field");
  if (f == SL2_SRC_GRAY_RING ? (src->width != 0 || src->height != 0)
                             : (src->width < 1 || src->height < 1 || src->width > SL2_MAX_SOURCE_DIM ||
                                src->height > SL2_MAX_SOURCE_DIM))
    return fail(c, SL2_ERR_ARG,
                "sl2_set_stream_source: size must be 0 x 0 for the default source, else in [1, SL2_MAX_SOURCE_DIM]");
  if (f == SL2_SRC_UYVY && (src->width & 1))
    return fail(c, SL2_ERR_ARG, "sl2_set_stream_source: a UYVY frame has an even width");
  std::vector<sl2_stream_source> srcs = c->srcs;
  srcs[s] = *src;
  return install_sources(c, srcs);
}

int sl2_get_stream_source(sl2_ctx *c, int32_t s, sl2_stream_source *src) {
  if (bad_stream(c, s) || !src) return fail(c, SL2_ERR_ARG, "sl2_get_stream_source: bad argument");
  *src = c->srcs[s];
  return SL2_OK;
}

int sl2_frame_set_layout(sl2_ctx *c, size_t *offsets) {
  enter(c);
  if (!c || !offsets) return fail(c, SL2_ERR_ARG, "sl2_frame_set_layout: bad argument");
  std::copy(c->layout.begin(), c->layout.end(), offsets);
  return SL2_OK;
}

int sl2_set_frame(sl2_ctx *c, int32_t s, int32_t slot, const uint8_t *gray, size_t stride) {
  if (bad_stream(c, s) || bad_slot(c, slot) || !gray) return fail(c, SL2_ERR_ARG, "sl2_set_frame: bad argument");
  const Sl2Dev &d = c->d;
  if (c->srcs[s].format != SL2_SRC_GRAY_RING) {  // the raw frame to the slot's staging, then its conversion
    int j = 0;
    while (c->src_rows[j].stream != s) ++j;
    const Sl2Source &r = c->src_rows[j];
    const size_t rb = (size_t)r.sw * sl2_source_bpp(r.format);
    CU_TRY(c, cudaMemcpy2DAsync(source_stage(c, slot) + r.off, rb, gray, stride, rb, r.sh, cudaMemcpyHostToDevice,
                                c->stream));
    CU_TRY(c, ingest(c, slot, j, 1, queue(c)));
  } else {
    uint8_t *dst = d.frames + ((size_t)slot * d.B + s) * d.H * d.pitch;
    const sl2_stream_config &sc = c->cams[s];  // the stream's image, top-left of its block
    CU_TRY(c, cudaMemcpy2DAsync(dst, d.pitch, gray, stride, sc.width, sc.height, cudaMemcpyHostToDevice, c->stream));
  }
  CU_TRY(c, cudaEventRecord(c->ev_slot[slot].cmp.get(), c->stream));  // slot busy until the copy has landed
  return SL2_OK;
}

static int set_frames_any(sl2_ctx *c, int32_t slot, const uint8_t *gray, cudaMemcpyKind kind) {
  enter(c);
  if (!c || bad_slot(c, slot) || !gray) return fail(c, SL2_ERR_ARG, "sl2_set_frames: bad argument");
  CU_TRY(c, copy_slot_frames(c, slot, gray, kind, queue(c)));
  CU_TRY(c, cudaEventRecord(c->ev_slot[slot].cmp.get(), c->stream));  // slot busy until the copy has landed
  return SL2_OK;
}
int sl2_set_frames(sl2_ctx *c, int32_t slot, const uint8_t *gray) {
  return set_frames_any(c, slot, gray, cudaMemcpyHostToDevice);
}
int sl2_set_frames_dev(sl2_ctx *c, int32_t slot, const uint8_t *gray_dev) {
  return set_frames_any(c, slot, gray_dev, cudaMemcpyDeviceToDevice);
}

}  // extern "C"
