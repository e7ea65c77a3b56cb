// detect.cu — Shi-Tomasi "best patch" detector on sm_90a (SURVEY.md §8(f) row N3).
//
// Replaces MonoSLAM::find_best_patch_inside_region + find_eigenvalues (monoslam.cpp:1070-1205):
// the smaller eigenvalue of the BOXSIZE x BOXSIZE gradient structure tensor, maximised over a
// region, first maximum in (v-major, u-minor) scan order (strict `>` against evbest = 0).
//
// The reference keeps running double sums of gx*gx etc. with gx = (I[c+1]-I[c-1])/2.0.  Those are
// multiples of 0.25 far below 2^53, so every running sum is EXACT whatever the order; the kernel
// therefore forms the exact int32 sums Sxx = sum dx^2 ... per position directly and converts with
// one exact multiply by 0.25.  The eigenvalue formula is evaluated op for op with never-fused
// __d*_rn (same bits as the x86-64 SSE2 build).
//
// Layout: one CTA per 32 x 32 tile of candidate positions of one region (grid = tiles x regions, any number of
// regions of one frame per launch).  The CTA stages the (32 + BOX + 1)^2 pixel window once, forms the three
// gradient products per pixel once, sums them along rows (sliding window of BOX, one thread per row segment) and
// then along columns: (BOX + BOX) adds per position instead of the BOX^2 gradient evaluations and 3 BOX^2
// multiply-adds of a per-position scan, and each pixel is read from global memory once per tile instead of
// once per position that covers it.  A second small kernel takes the best of the tiles of each region.
// Entry point: sl2_find_best_patch.
#include "sl2_context.cuh"

using namespace sl2;

namespace {

struct DBest {
  double ev;
  int idx;
};

__device__ __forceinline__ void dconsider(DBest &b, double ev, int idx) {
  // strict `eval2 > *evbest` in scan order: larger wins, equal keeps the earlier position
  if (ev > 0.0 && (ev > b.ev || (ev == b.ev && idx < b.idx))) {
    b.ev = ev;
    b.idx = idx;
  }
}

constexpr int DT = 32;        // tile of candidate positions (DT x DT)
constexpr int DTHREADS = 256;

// monoslam.cpp:1083-1090: the scan window of a region after clipping to where the box fits in the stream's W x H image
__device__ __forceinline__ void clip_region(int W, int H, const int *reg, int HALF, int &us, int &vs, int &uf,
                                            int &vf) {
  us = reg[0], vs = reg[1], uf = reg[2], vf = reg[3];
  if (us < HALF + 1) us = HALF + 1;
  if (uf > W - HALF - 1) uf = W - HALF - 1;
  if (vs < HALF + 1) vs = HALF + 1;
  if (vf > H - HALF - 1) vf = H - HALF - 1;
}

template <int BOX>
__global__ void __launch_bounds__(DTHREADS) detect_tiles_kernel(const Sl2Dev d, int stream, int slot,
                                                               const int *regions, int max_tiles,
                                                               double *part_ev, int *part_idx) {
  constexpr int HALF = (BOX - 1) / 2;
  constexpr int IW = DT + BOX + 1;   // staged pixels per row / rows
  constexpr int GW = DT + BOX - 1;   // pixels with a gradient: the union of the boxes of the tile
  __shared__ uint8_t s_img[IW][IW + 3];
  __shared__ int s_g[3][GW][GW + 1];   // dx*dx, dy*dy, dx*dy per pixel
  __shared__ int s_h[3][GW][DT + 1];   // the same summed over BOX pixels along the row, per position column
  // the reduction arrays reuse the gradient products (dead by then): the static 48 KB limit
  double *s_ev = reinterpret_cast<double *>(&s_g[0][0][0]);
  int *s_idx = reinterpret_cast<int *>(s_ev + DTHREADS);
  static_assert(sizeof(int) * GW * (GW + 1) >= DTHREADS * (sizeof(double) + sizeof(int)), "reduction scratch");
  const int job = blockIdx.y, tile = blockIdx.x, tid = threadIdx.x;
  const int Ws = stream_width(d.cams[stream]), Hs = stream_height(d.cams[stream]);
  int us, vs, uf, vf;
  clip_region(Ws, Hs, regions + job * 4, HALF, us, vs, uf, vf);
  DBest best = {0.0, 0x7fffffff};
  const int RW = uf - us, RH = vf - vs;
  const int tiles_x = RW > 0 ? (RW + DT - 1) / DT : 0, tiles_y = RH > 0 ? (RH + DT - 1) / DT : 0;
  if (tile < tiles_x * tiles_y) {  // (an empty region has no tiles: monoslam.cpp:1093-1098)
    const int u0 = us + (tile % tiles_x) * DT, v0 = vs + (tile / tiles_x) * DT;
    const uint8_t *img = d.frames + ((size_t)slot * d.B + stream) * d.H * d.pitch;
    // pixel window: rows v0-HALF-1 .. v0+DT+HALF, columns likewise (clamped to the stream's image: positions past
    // the region are dropped)
    for (int e = tid; e < IW * IW; e += DTHREADS) {
      const int r = e / IW, c = e - r * IW;
      const int y = min(v0 - HALF - 1 + r, Hs - 1), x = min(u0 - HALF - 1 + c, Ws - 1);
      s_img[r][c] = __ldg(img + (size_t)y * d.pitch + x);
    }
    __syncthreads();
    for (int e = tid; e < GW * GW; e += DTHREADS) {
      const int r = e / GW, c = e - r * GW;  // pixel (v0-HALF+r, u0-HALF+c) = s_img[r+1][c+1]
      const int dx = (int)s_img[r + 1][c + 2] - (int)s_img[r + 1][c];
      const int dy = (int)s_img[r + 2][c + 1] - (int)s_img[r][c + 1];
      s_g[0][r][c] = dx * dx;
      s_g[1][r][c] = dy * dy;
      s_g[2][r][c] = dx * dy;
    }
    __syncthreads();
    // row sums: thread = (product, row, segment of 8 position columns); sliding window along the row
    for (int e = tid; e < 3 * GW * (DT / 8); e += DTHREADS) {
      const int seg = e % (DT / 8), r = (e / (DT / 8)) % GW, q = e / ((DT / 8) * GW);
      const int *g = s_g[q][r] + seg * 8;
      int acc = 0;
#pragma unroll
      for (int c = 0; c < BOX; ++c) acc += g[c];
      s_h[q][r][seg * 8] = acc;
#pragma unroll
      for (int k = 1; k < 8; ++k) {
        acc += g[BOX - 1 + k] - g[k - 1];
        s_h[q][r][seg * 8 + k] = acc;
      }
    }
    __syncthreads();
    // column sums and the eigenvalue: thread = position column tx, rows ty, ty+8, ty+16, ty+24
    const int tx = tid & 31, ty = tid >> 5;
#pragma unroll
    for (int k = 0; k < DT / 8; ++k) {
      const int py = ty + 8 * k;
      const int u = u0 + tx, v = v0 + py;
      if (u < uf && v < vf) {
        int Sxx = 0, Syy = 0, Sxy = 0;
#pragma unroll
        for (int r = 0; r < BOX; ++r) {
          Sxx += s_h[0][py + r][tx];
          Syy += s_h[1][py + r][tx];
          Sxy += s_h[2][py + r][tx];
        }
        // TSgxsq = Sxx/4 etc. (exact); find_eigenvalues(A = TSgxsq, B = TSgxgy, C = TSgysq)
        const double A = mul_((double)Sxx, 0.25), B = mul_((double)Sxy, 0.25), C = mul_((double)Syy, 0.25);
        const double t1 = add_(A, C);
        const double BB = sqrt_(sub_(mul_(t1, t1), mul_(4.0, sub_(mul_(A, C), mul_(B, B)))));
        const double eval2 = div_(sub_(t1, BB), 2.0);
        dconsider(best, eval2, (v - vs) * RW + (u - us));
      }
    }
  }
  __syncthreads();  // (uniform: `tile` is per CTA) the row-sum pass has read s_g
  s_ev[tid] = best.ev;
  s_idx[tid] = best.idx;
  __syncthreads();
  for (int o = DTHREADS / 2; o > 0; o >>= 1) {
    if (tid < o) {
      DBest a = {s_ev[tid], s_idx[tid]};
      dconsider(a, s_ev[tid + o], s_idx[tid + o]);
      s_ev[tid] = a.ev;
      s_idx[tid] = a.idx;
    }
    __syncthreads();
  }
  if (tid == 0) {
    part_ev[(size_t)job * max_tiles + tile] = s_ev[0];
    part_idx[(size_t)job * max_tiles + tile] = s_idx[0];
  }
}

__global__ void __launch_bounds__(128) detect_reduce_kernel(const Sl2Dev d, int stream, const int *regions, int half,
                                                            int max_tiles, const double *part_ev,
                                                            const int *part_idx, int *out_uv, double *out_ev) {
  __shared__ double s_ev[128];
  __shared__ int s_idx[128];
  const int job = blockIdx.x, tid = threadIdx.x;
  int us, vs, uf, vf;
  clip_region(stream_width(d.cams[stream]), stream_height(d.cams[stream]), regions + job * 4, half, us, vs, uf, vf);
  DBest best = {0.0, 0x7fffffff};
  for (int t = tid; t < max_tiles; t += 128)
    dconsider(best, part_ev[(size_t)job * max_tiles + t], part_idx[(size_t)job * max_tiles + t]);
  s_ev[tid] = best.ev;
  s_idx[tid] = best.idx;
  __syncthreads();
  for (int o = 64; o > 0; o >>= 1) {
    if (tid < o) {
      DBest a = {s_ev[tid], s_idx[tid]};
      dconsider(a, s_ev[tid + o], s_idx[tid + o]);
      s_ev[tid] = a.ev;
      s_idx[tid] = a.idx;
    }
    __syncthreads();
  }
  if (tid == 0) {
    if (vs >= vf || us >= uf) {  // monoslam.cpp:1093-1098
      out_uv[job * 2 + 0] = us;
      out_uv[job * 2 + 1] = vs;
      out_ev[job] = 0.0;
    } else {
      const int RW = uf - us;
      if (s_idx[0] != 0x7fffffff) {
        out_uv[job * 2 + 0] = us + s_idx[0] % RW;
        out_uv[job * 2 + 1] = vs + s_idx[0] / RW;
      } else {
        out_uv[job * 2 + 0] = -1;  // nothing beat evbest = 0: the reference leaves *ubest/*vbest alone
        out_uv[job * 2 + 1] = -1;
      }
      out_ev[job] = s_ev[0];
    }
  }
}

// bytes of device scratch the launch needs for n regions of a W x H frame (per-tile partial results)
size_t sl2_detect_scratch_bytes(const Sl2Dev &d, int n) {
  const int max_tiles = ((d.W + DT - 1) / DT) * ((d.H + DT - 1) / DT);
  return (size_t)n * max_tiles * (sizeof(double) + sizeof(int)) + 16;
}

cudaError_t sl2_launch_detect(const Sl2Dev &d, int stream, int slot, int n, const int *regions_dev,
                              int *out_uv_dev, double *out_ev_dev, void *scratch_dev, Sl2Queue q) {
  if (n <= 0) return cudaSuccess;
  const int max_tiles = ((d.W + DT - 1) / DT) * ((d.H + DT - 1) / DT);
  double *part_ev = reinterpret_cast<double *>(scratch_dev);
  int *part_idx = reinterpret_cast<int *>(part_ev + (size_t)n * max_tiles);
  const dim3 grid(max_tiles, n);
  const cudaError_t e = sl2_with_box(d.box, [&](auto box) {
    return sl2_launch_kernel(detect_tiles_kernel<decltype(box)::value>, grid, dim3(DTHREADS), 0, q, false, d, stream,
                             slot, regions_dev, max_tiles, part_ev, part_idx);
  });
  if (e != cudaSuccess) return e;
  return sl2_launch_kernel(detect_reduce_kernel, dim3(n), dim3(128), 0, q, false, d, stream, regions_dev,
                           (d.box - 1) / 2, max_tiles, part_ev, part_idx, out_uv_dev, out_ev_dev);
}

}  // namespace

extern "C" {

int sl2_find_best_patch(sl2_ctx *c, int32_t s, int32_t slot, int32_t n, const int32_t *regions,
                        int32_t *ubest, int32_t *vbest, double *evbest) {
  if (bad_stream(c, s) || bad_slot(c, slot) || n < 0 || (n && (!regions || !evbest)))
    return fail(c, SL2_ERR_ARG, "sl2_find_best_patch: bad argument");
  if (n == 0) return SL2_OK;
  Stage rg{STAGE_IN, 16 * (size_t)n, regions}, uv{STAGE_OUT, 8 * (size_t)n}, ev{STAGE_OUT, 8 * (size_t)n},
      scratch{STAGE_DEV, sl2_detect_scratch_bytes(c->d, n)};
  const int rc = staged_call(c, {&rg, &uv, &ev, &scratch}, [] {}, [&] {
    CU_TRY(c, sl2_launch_detect(c->d, s, slot, n, rg.dev<int>(), uv.dev<int>(), ev.dev<double>(), scratch.d, queue(c)));
    return SL2_OK;
  });
  if (rc) return rc;
  for (int i = 0; i < n; ++i) {
    evbest[i] = ev.host<double>()[i];
    if (uv.host<int>()[2 * i] >= 0) {
      if (ubest) ubest[i] = uv.host<int>()[2 * i];
      if (vbest) vbest[i] = uv.host<int>()[2 * i + 1];
    }
  }
  return SL2_OK;
}

}  // extern "C"
