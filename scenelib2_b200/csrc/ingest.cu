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
#include "sl2_common.cuh"

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

}  // namespace

cudaError_t sl2_launch_source_write(Sl2Source *table, const Sl2SourceChunk &chunk, Sl2Queue q) {
  return sl2_launch_kernel(source_write_kernel, dim3(1), dim3(SL2_SOURCE_CHUNK), 0, q, false, table, chunk);
}

cudaError_t sl2_launch_ingest(const Sl2Dev &d, const Sl2Source *table, int base, int cnt, int max_dh,
                              int max_row_bytes, const uint8_t *stage_slot, int slot, Sl2Queue q) {
  if (cnt <= 0) return cudaSuccess;
  const int row_cap = ((max_row_bytes + 15) & ~15) + 16;  // one raw row at any 16-byte misalignment
  const dim3 grid((max_dh + INGEST_ROWS - 1) / INGEST_ROWS, cnt);
  uint8_t *ring_slot = d.frames + (size_t)slot * d.B * d.H * d.pitch;
  return sl2_launch_kernel(ingest_kernel, grid, dim3(INGEST_THREADS), 2 * (size_t)row_cap, q, false, table, base,
                           stage_slot, ring_slot, d.H, d.pitch, row_cap);
}
