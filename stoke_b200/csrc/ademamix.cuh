// ademamix.cuh -- AdEMAMix's per-step scalars, shared by the fp32 step's prologue (k2_optim.cu) and the 8-bit step's
// (k2_optim8bit.cu), so both form the same four numbers from the same double arithmetic.
#pragma once

#include "common.cuh"

namespace stk {

// apple/ml-ademamix's half-life map of the beta3 warm-up: f(b) = log(0.5) / log(b + 1e-8) - 1
__device__ __forceinline__ double ademamix_f(double b) {
  return __dadd_rn(__ddiv_rn(log(0.5), log(__dadd_rn(b, 1e-8))), -1.0);
}

// AdEMAMix.step's per-step scalars of step t, in python doubles and python's order (the explicit roundings keep nvcc
// from contracting a * b + c into one DFMA, which python does not do):  {1 / bc1, 1 / sqrt(bc2), alpha_t, 1 - beta3_t}.
// beta3_t itself, when given, receives fp32(beta3_t).
__device__ __forceinline__ float4 ademamix_scalars(double beta1, double beta2, const stk_ademamix_hyper_t& h, double t,
                                                   float* beta3_out = nullptr) {
  const double bc1 = __dadd_rn(1.0, -pow(beta1, t));
  const double bc2 = __dadd_rn(1.0, -pow(beta2, t));
  double alpha_t = h.alpha;
  if (h.alpha_warmup > 0 && t < (double)h.alpha_warmup) alpha_t = __dmul_rn(__ddiv_rn(t, (double)h.alpha_warmup), h.alpha);
  double beta3_t = h.beta3;
  if (h.beta3_warmup > 0 && t < (double)h.beta3_warmup) {
    const double a = __ddiv_rn(t, (double)h.beta3_warmup);
    const double x = __dadd_rn(__dmul_rn(__dadd_rn(1.0, -a), ademamix_f(beta1)), __dmul_rn(a, ademamix_f(h.beta3)));
    beta3_t = pow(0.5, __ddiv_rn(1.0, __dadd_rn(x, 1.0)));   // f_inv(x) = 0.5 ** (1 / (x + 1))
  }
  if (beta3_out != nullptr) *beta3_out = (float)beta3_t;
  return make_float4((float)__ddiv_rn(1.0, bc1), (float)__ddiv_rn(1.0, __dsqrt_rn(bc2)), (float)alpha_t,
                     (float)__dadd_rn(1.0, -beta3_t));
}

}  // namespace stk
