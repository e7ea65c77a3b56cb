// dmma_rate.cu — sustained FP64 tensor-core rate of the four mma.sync f64 shapes sm_90 has, and a check of their
// fragment layouts against a CPU product.
//
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o dmma_rate tools/dmma_rate.cu && ./dmma_rate
//
// For each shape (m8n8k4, m16n8k4, m16n8k8, m16n8k16) it times a grid of 4 CTAs x 256 threads per SM, every warp
// running 8 independent accumulator chains, in four cases:
//   reg      A and B fragments in registers (the pipe's own rate)
//   smem/1   a fresh A fragment read from shared memory for every MMA: 1 B of shared memory per FMA, what the
//            upd_solve trailing update and the upd_syrk slab loop read (with the slab fill) per FMA
//   smem/2   each A fragment read serves 2 MMAs (0.5 B/FMA)
//   smem/4   each A fragment read serves 4 MMAs (0.25 B/FMA)
// The rate is 2 * M * N * K * (MMAs) / time (CUDA events, best of 3 launches after a warm-up launch).  The program
// exits with status 1 if a layout check fails.
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <cuda_runtime.h>

#define CK(x)                                                                              \
  do {                                                                                     \
    cudaError_t e_ = (x);                                                                  \
    if (e_ != cudaSuccess) {                                                               \
      std::fprintf(stderr, "%s:%d %s\n", __FILE__, __LINE__, cudaGetErrorString(e_));      \
      std::exit(2);                                                                        \
    }                                                                                      \
  } while (0)

// KA / KB: doubles per lane of the A / B fragment; M, K: shape (N = 8)
template <int SH> struct Shape;
template <> struct Shape<0> { static constexpr int M = 8, K = 4, KA = 1, KB = 1; static constexpr const char *name = "m8n8k4"; };
template <> struct Shape<1> { static constexpr int M = 16, K = 4, KA = 2, KB = 1; static constexpr const char *name = "m16n8k4"; };
template <> struct Shape<2> { static constexpr int M = 16, K = 8, KA = 4, KB = 2; static constexpr const char *name = "m16n8k8"; };
template <> struct Shape<3> { static constexpr int M = 16, K = 16, KA = 8, KB = 4; static constexpr const char *name = "m16n8k16"; };

// c: 2 (m8) or 4 (m16) accumulators
template <int SH>
__device__ __forceinline__ void mma(double *c, const double *a, const double *b) {
  if constexpr (SH == 0) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                 : "+d"(c[0]), "+d"(c[1]) : "d"(a[0]), "d"(b[0]));
  } else if constexpr (SH == 1) {
    asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a[0]), "d"(a[1]), "d"(b[0]));
  } else if constexpr (SH == 2) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                 "{%0,%1,%2,%3};"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                 : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
  } else {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
                 "{%12,%13,%14,%15}, {%0,%1,%2,%3};"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                 : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
                   "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
  }
}

// ---- layout check: one warp, A (M x K) and B (K x 8) row-major in global memory -------------------------------
// A fragment element i of lane (g = lane/4, t = lane%4): row g + 8 (i % 2), column t + 4 (i / 2)  (m8n8k4: row g, col t)
// B fragment element i: row t + 4 i, column g.   C element e: row g + 8 (e / 2), column 2 t + e % 2.
template <int SH>
__global__ void layout_kernel(const double *A, const double *B, double *C) {
  using S = Shape<SH>;
  const int lane = threadIdx.x, g = lane >> 2, t = lane & 3;
  double a[8], b[4], c[4] = {0.0, 0.0, 0.0, 0.0};
  for (int i = 0; i < S::KA; ++i) a[i] = A[(g + 8 * (i % 2)) * S::K + t + 4 * (i / 2)];
  if (SH == 0) a[0] = A[g * S::K + t];
  for (int i = 0; i < S::KB; ++i) b[i] = B[(t + 4 * i) * 8 + g];
  mma<SH>(c, a, b);
  for (int e = 0; e < (S::M == 16 ? 4 : 2); ++e) C[(g + 8 * (e / 2)) * 8 + 2 * t + e % 2] = c[e];
}

template <int SH>
bool check_layout() {
  using S = Shape<SH>;
  double hA[16 * 16], hB[16 * 8], hC[16 * 8], ref[16 * 8];
  for (int i = 0; i < S::M * S::K; ++i) hA[i] = (double)((i * 37) % 23 - 11);
  for (int i = 0; i < S::K * 8; ++i) hB[i] = (double)((i * 11) % 17 - 8);
  for (int r = 0; r < S::M; ++r)
    for (int c = 0; c < 8; ++c) {
      double s = 0.0;
      for (int k = 0; k < S::K; ++k) s += hA[r * S::K + k] * hB[k * 8 + c];
      ref[r * 8 + c] = s;
    }
  double *dA, *dB, *dC;
  CK(cudaMalloc(&dA, sizeof hA));
  CK(cudaMalloc(&dB, sizeof hB));
  CK(cudaMalloc(&dC, sizeof hC));
  CK(cudaMemcpy(dA, hA, sizeof hA, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dB, hB, sizeof hB, cudaMemcpyHostToDevice));
  layout_kernel<SH><<<1, 32>>>(dA, dB, dC);
  CK(cudaGetLastError());
  CK(cudaMemcpy(hC, dC, sizeof hC, cudaMemcpyDeviceToHost));
  CK(cudaFree(dA));
  CK(cudaFree(dB));
  CK(cudaFree(dC));
  bool ok = true;
  for (int i = 0; i < S::M * 8; ++i) ok = ok && hC[i] == ref[i];  // small integers: exact
  return ok;
}

// ---- rate kernel ---------------------------------------------------------------------------------------------
constexpr int CHAINS = 8;
constexpr int THREADS = 256;
// MODE 0: registers; MODE r > 0: an A fragment from shared memory serves r MMAs (r different B fragments)
template <int SH, int MODE>
__global__ void __launch_bounds__(THREADS) rate_kernel(int iters, double *out) {
  using S = Shape<SH>;
  __shared__ double sa[2048];
  const int lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < 2048; i += THREADS) sa[i] = 1e-3 * (i % 7);
  __syncthreads();
  double c[CHAINS][4], a[S::KA], b[CHAINS][S::KB];
#pragma unroll
  for (int q = 0; q < CHAINS; ++q) {
    c[q][0] = c[q][1] = c[q][2] = c[q][3] = 0.0;
#pragma unroll
    for (int i = 0; i < S::KB; ++i) b[q][i] = 1e-3 * (lane + q + i);
  }
#pragma unroll
  for (int i = 0; i < S::KA; ++i) a[i] = 1e-3 * (lane - i);
  // the shared-memory A fragments walk a 2048-double window, conflict-free (32 consecutive doubles per read)
  int off = (threadIdx.x >> 5) * 64 + lane;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int q = 0; q < CHAINS; ++q) {
      if (MODE > 0 && q % MODE == 0) {
#pragma unroll
        for (int i = 0; i < S::KA; ++i) a[i] = sa[(off + 32 * i) & 2047];
        off += 32 * S::KA;
      }
      mma<SH>(c[q], a, b[q]);
    }
  }
  double s = 0.0;
#pragma unroll
  for (int q = 0; q < CHAINS; ++q) s += c[q][0] + c[q][1] + c[q][2] + c[q][3];
  if (s == 12345.678) out[threadIdx.x] = s;  // keeps the chains alive
}

template <int SH, int MODE>
double rate(int nsm, double *out) {
  using S = Shape<SH>;
  const int blocks = 4 * nsm, iters = 4096;
  rate_kernel<SH, MODE><<<blocks, THREADS>>>(iters, out);  // warm-up
  CK(cudaGetLastError());
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  float best = 1e30f;
  for (int r = 0; r < 3; ++r) {
    CK(cudaEventRecord(e0));
    rate_kernel<SH, MODE><<<blocks, THREADS>>>(iters, out);
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    if (ms < best) best = ms;
  }
  CK(cudaEventDestroy(e0));
  CK(cudaEventDestroy(e1));
  const double mmas = (double)blocks * (THREADS / 32) * iters * CHAINS;
  return 2.0 * S::M * 8 * S::K * mmas / (best * 1e-3) / 1e12;
}

template <int SH>
bool row(int nsm, double *out) {
  const bool ok = check_layout<SH>();
  std::printf("%-9s layout %-4s  reg %6.2f   smem/1 %6.2f   smem/2 %6.2f   smem/4 %6.2f  TFLOP/s\n", Shape<SH>::name,
              ok ? "ok" : "BAD", rate<SH, 0>(nsm, out), rate<SH, 1>(nsm, out), rate<SH, 2>(nsm, out),
              rate<SH, 4>(nsm, out));
  return ok;
}

int main() {
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  std::printf("%s, %d SMs\n", prop.name, prop.multiProcessorCount);
  double *out;
  CK(cudaMalloc(&out, THREADS * sizeof(double)));
  bool ok = row<0>(prop.multiProcessorCount, out);
  ok = row<1>(prop.multiProcessorCount, out) && ok;
  ok = row<2>(prop.multiProcessorCount, out) && ok;
  ok = row<3>(prop.multiProcessorCount, out) && ok;
  CK(cudaFree(out));
  return ok ? 0 : 1;
}
