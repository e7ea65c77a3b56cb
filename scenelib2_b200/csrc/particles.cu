// particles.cu — depth particles of partially-initialised features (SURVEY N2): the re-weighting of
// sl2_measure_partial_features / sl2_measure_particles.  Their prediction (particle_predict_kernel) is in ekf.cu, with
// the measurement models it shares with map features.
//   particle_kernel   MonoSLAM::update_partially_initialised_feature_probabilities (monoslam.cpp:1447-1493, body for
//                     one FeatureInitInfo) + FeatureInitInfo::normalise_particle_vector_and_calculate_cumulative /
//                     prune_particle_vector / calculate_mean_and_covariance (feature_init_info.cpp:95-172), after the
//                     SMOE kernels (smoe.cu), on the match positions they left in device memory; one CTA per feature.
#include "sl2_common.cuh"

namespace {

// One CTA.  The likelihoods are independent (one thread per particle); the normalisation sums are
// order dependent in FP64, so one thread adds them in particle order like the reference's loops.
__global__ void __launch_bounds__(128) particle_kernel(int Kmax, const int *__restrict__ Kf,
                                                       const double *__restrict__ h,
                                                       const double *__restrict__ sinv3,
                                                       const double *__restrict__ detS,
                                                       const double *__restrict__ lambda,
                                                       const int *__restrict__ z_uv,
                                                       const uint8_t *__restrict__ found, double prune_threshold,
                                                       double *prob, uint8_t *keep, double *cumulative,
                                                       double *mean_var, int *left_out) {
  {  // feature blockIdx.x: its K particles at offset blockIdx.x * Kmax of every array
    const size_t o = (size_t)blockIdx.x * Kmax;
    h += 2 * o, sinv3 += 3 * o, detS += o, lambda += o, z_uv += 2 * o, found += o;
    prob += o, keep += o, cumulative += o, mean_var += 2 * blockIdx.x, left_out += blockIdx.x;
  }
  const int K = Kf[blockIdx.x];
  for (int k = threadIdx.x; k < K; k += blockDim.x) {  // monoslam.cpp:1456-1478
    double likelihood = 0.0;
    if (found[k]) {
      const double nu0 = sub_((double)z_uv[2 * k], h[2 * k]), nu1 = sub_((double)z_uv[2 * k + 1], h[2 * k + 1]);
      const double r0 = add_(mul_(sinv3[3 * k], nu0), mul_(sinv3[3 * k + 1], nu1));
      const double r1 = add_(mul_(sinv3[3 * k + 1], nu0), mul_(sinv3[3 * k + 2], nu1));
      const double q = add_(mul_(nu0, r0), mul_(nu1, r1));
      // 1 / sqrt(2 pi det S) * exp(-q / 2); device exp is within 1 ulp of the correctly rounded value
      likelihood = mul_(div_(1.0, sqrt_(mul_(6.283185307179586476925286766559, detS[k]))), exp(mul_(-0.5, q)));
    }
    prob[k] = mul_(prob[k], likelihood);
    keep[k] = 1;
    cumulative[k] = 0.0;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  auto normalise = [&]() -> bool {  // feature_init_info.cpp:95-119
    double total = 0.0;
    for (int k = 0; k < K; ++k)
      if (keep[k]) total = add_(total, prob[k]);
    if (total == 0.0) return false;
    double cum = 0.0;
    for (int k = 0; k < K; ++k)
      if (keep[k]) {
        const double p = div_(prob[k], total);
        prob[k] = p;
        cumulative[k] = add_(cum, p);
        cum = add_(cum, p);
      }
    return true;
  };
  mean_var[0] = mean_var[1] = 0.0;
  if (!normalise()) {  // every match failed: the reference deletes the feature (monoslam.cpp:1486-1490)
    for (int k = 0; k < K; ++k) keep[k] = 0;
    *left_out = 0;
    return;
  }
  const double thr = div_(prune_threshold, (double)K);  // feature_init_info.cpp:128
  int left = 0;
  for (int k = 0; k < K; ++k) {
    if (prob[k] < thr) {
      keep[k] = 0;
      cumulative[k] = 0.0;
    } else {
      ++left;
    }
  }
  normalise();
  double mean = 0.0, e2 = 0.0;  // feature_init_info.cpp:152-172, scalar lambda
  for (int k = 0; k < K; ++k)
    if (keep[k]) {
      mean = add_(mean, mul_(prob[k], lambda[k]));
      e2 = add_(e2, mul_(prob[k], mul_(lambda[k], lambda[k])));
    }
  mean_var[0] = mean;
  mean_var[1] = sub_(e2, mul_(mean, mean));
  *left_out = left;
}

}  // namespace

// F features, Kmax = stride between features in every per-particle array, K_dev[f] particles used
cudaError_t sl2_launch_particles(int F, int Kmax, const int *K_dev, const double *h, const double *sinv3,
                                 const double *detS, const double *lambda, const int *z_uv, const uint8_t *found,
                                 double prune_threshold, double *prob, uint8_t *keep, double *cumulative,
                                 double *mean_var, int *left_out, Sl2Queue q) {
  if (F <= 0) return cudaSuccess;
  return sl2_launch_kernel(particle_kernel, dim3(F), dim3(128), 0, q, false, Kmax, K_dev, h, sinv3, detS, lambda, z_uv,
                           found, prune_threshold, prob, keep, cumulative, mean_var, left_out);
}
