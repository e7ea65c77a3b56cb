// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the shipped product path.
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
// legs may load anything under oracle/.
//
// Minimal column-major FP64 dense algebra standing in for the Eigen3 calls on the
// SceneLib2 hot path (Eigen3 is an un-vendored dependency of the reference, version
// unpinned: CMakeModules/FindEigen3.cmake:17-30, README:71-72).
//
// Rules (SURVEY.md §8(c)): plain C++17, column-major, FP64, products evaluated in the
// association order the reference writes them, inner-product accumulation in ascending k,
// standard lower Cholesky, triangular inverse by forward substitution, compiled with
// -O3 -ffp-contract=off and no -march (the reference's Release build has no FMA).
// PARITY UNPINNED at the last ulp versus a true Eigen3 build: Eigen's blocked/vectorised
// accumulation order cannot be reproduced without Eigen, and the reference ships no
// golden outputs.  The 1e-5 relative tolerance of the north star absorbs this.
// Everything else -- formulas, control flow, operation order -- is pinned to the reference's own
// sources compiled against oracle/stubs_arith (oracle/_ref/libsl2refmodels.so, tests/test_oracle_ref.py).
#pragma once
#include <cmath>
#include <cstddef>
#include <cstring>
#include <vector>

namespace sl2o {

struct Mat {
  int r = 0, c = 0;
  std::vector<double> a;
  Mat() {}
  Mat(int rows, int cols) : r(rows), c(cols), a((size_t)rows * cols, 0.0) {}
  double &operator()(int i, int j) { return a[(size_t)i + (size_t)j * r]; }
  double operator()(int i, int j) const { return a[(size_t)i + (size_t)j * r]; }
  void zero() { std::fill(a.begin(), a.end(), 0.0); }
  void identity() {
    zero();
    for (int i = 0; i < r && i < c; ++i) (*this)(i, i) = 1.0;
  }
  double *col(int j) { return a.data() + (size_t)j * r; }
  const double *col(int j) const { return a.data() + (size_t)j * r; }
};

typedef std::vector<double> Vec;

// C = A * B ; every C(i,j) is accumulated over k ascending starting from 0.0.
// Loop order j-k-i keeps the inner loop contiguous (column-major) so gcc -O3 can use
// SSE2 without changing the per-element summation order.
inline Mat mul(const Mat &A, const Mat &B) {
  Mat C(A.r, B.c);
  const int M = A.r, K = A.c, N = B.c;
  for (int j = 0; j < N; ++j) {
    double *cj = C.col(j);
    for (int k = 0; k < K; ++k) {
      const double b = B(k, j);
      const double *ak = A.col(k);
      for (int i = 0; i < M; ++i) cj[i] += ak[i] * b;
    }
  }
  return C;
}

// C = A * B^T
inline Mat mul_nt(const Mat &A, const Mat &B) {
  Mat C(A.r, B.r);
  const int M = A.r, K = A.c, N = B.r;
  for (int j = 0; j < N; ++j) {
    double *cj = C.col(j);
    for (int k = 0; k < K; ++k) {
      const double b = B(j, k);
      const double *ak = A.col(k);
      for (int i = 0; i < M; ++i) cj[i] += ak[i] * b;
    }
  }
  return C;
}

// C = A^T * B
inline Mat mul_tn(const Mat &A, const Mat &B) {
  Mat C(A.c, B.c);
  const int M = A.c, K = A.r, N = B.c;
  for (int j = 0; j < N; ++j) {
    const double *bj = B.col(j);
    for (int i = 0; i < M; ++i) {
      const double *ai = A.col(i);
      double s = 0.0;
      for (int k = 0; k < K; ++k) s += ai[k] * bj[k];
      C(i, j) = s;
    }
  }
  return C;
}

inline Vec mul(const Mat &A, const Vec &x) {
  Vec y((size_t)A.r, 0.0);
  for (int k = 0; k < A.c; ++k) {
    const double b = x[k];
    const double *ak = A.col(k);
    for (int i = 0; i < A.r; ++i) y[i] += ak[i] * b;
  }
  return y;
}

inline Mat transpose(const Mat &A) {
  Mat T(A.c, A.r);
  for (int j = 0; j < A.c; ++j)
    for (int i = 0; i < A.r; ++i) T(j, i) = A(i, j);
  return T;
}

inline Mat add(const Mat &A, const Mat &B) {
  Mat C(A.r, A.c);
  for (size_t i = 0; i < A.a.size(); ++i) C.a[i] = A.a[i] + B.a[i];
  return C;
}

inline void add_inplace(Mat &A, const Mat &B) {
  for (size_t i = 0; i < A.a.size(); ++i) A.a[i] += B.a[i];
}

inline void sub_inplace(Mat &A, const Mat &B) {
  for (size_t i = 0; i < A.a.size(); ++i) A.a[i] -= B.a[i];
}

inline Mat block(const Mat &A, int i0, int j0, int rows, int cols) {
  Mat B(rows, cols);
  for (int j = 0; j < cols; ++j)
    for (int i = 0; i < rows; ++i) B(i, j) = A(i0 + i, j0 + j);
  return B;
}

inline void set_block(Mat &A, int i0, int j0, const Mat &B) {
  for (int j = 0; j < B.c; ++j)
    for (int i = 0; i < B.r; ++i) A(i0 + i, j0 + j) = B(i, j);
}

inline void set_block_transposed(Mat &A, int i0, int j0, const Mat &B) {
  for (int j = 0; j < B.c; ++j)
    for (int i = 0; i < B.r; ++i) A(i0 + j, j0 + i) = B(i, j);
}

// Standard lower Cholesky S = L L^T (stands in for Eigen::LLT<MatrixXd>::matrixL(),
// kalman.cpp:104-105, monoslam.cpp:371-372).  Only the lower triangle of S is read.
// A non-positive pivot propagates NaN exactly like an unchecked LLT would.
inline Mat cholesky_lower(const Mat &S) {
  const int n = S.r;
  Mat L(n, n);
  for (int j = 0; j < n; ++j) {
    double d = S(j, j);
    for (int k = 0; k < j; ++k) d -= L(j, k) * L(j, k);
    const double ljj = std::sqrt(d);
    L(j, j) = ljj;
    for (int i = j + 1; i < n; ++i) {
      double s = S(i, j);
      for (int k = 0; k < j; ++k) s -= L(i, k) * L(j, k);
      L(i, j) = s / ljj;
    }
  }
  return L;
}

// Inverse of a lower-triangular matrix by forward substitution, column by column
// (stands in for MatrixXd::inverse() applied to S_L, kalman.cpp:106, monoslam.cpp:373).
inline Mat lower_inverse(const Mat &L) {
  const int n = L.r;
  Mat X(n, n);
  for (int j = 0; j < n; ++j) {
    X(j, j) = 1.0 / L(j, j);
    for (int i = j + 1; i < n; ++i) {
      double s = 0.0;
      for (int k = j; k < i; ++k) s -= L(i, k) * X(k, j);
      X(i, j) = s / L(i, i);
    }
  }
  return X;
}

}  // namespace sl2o
