// bn_act.cu -- BatchNorm apply (+ residual add) + ReLU in one pass over a bf16 NHWC activation, for training-mode
// BatchNorm whose statistics torch has already reduced (stk_bn_act in include/stoke_b200.h).
//
// Purely elementwise.  Every rounding of the unfused torch sequence is kept, so the result is bit-identical to it:
//   y = bf16(w * (x - mean) * invstd + b)        batch_norm_transform_input_channels_last_kernel (FADD, FMUL, FFMA)
//   z = bf16(float(y) + float(r))                `out += identity` on bf16 (fp32 add, one rounding)
//   out = isnan(z) ? z : bf16(fmaxf(z, 0))       relu_ = clamp_min_(0), which keeps a NaN's bits
//   invstd = rsqrtf(var + eps)                   batch_norm_update_stats_and_invert
// Bytes per element: x read 2 + out write 2 (+ residual read 2).  The unfused chain moves 8 (15 with the residual).
#include <algorithm>

#include "common.cuh"
#include "ctx.cuh"

namespace stk {

constexpr int kBnThreads = 256;

__device__ __forceinline__ uint16_t bf16_bits(float f) { return __bfloat16_as_ushort(__float2bfloat16_rn(f)); }
__device__ __forceinline__ float bf16_val(uint16_t u) { return __uint_as_float(uint32_t(u) << 16); }

// Thread t owns channel group t % G (G = C / 8) and walks rows t / G, t / G + T / G, ...: T (the active thread count) is a
// multiple of G, so the per-channel parameters stay in registers for the whole loop.
template <bool kResidual>
__global__ void __launch_bounds__(kBnThreads) k_bn_act(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ r,
                                                      const float* __restrict__ mean, const float* __restrict__ var,
                                                      const __nv_bfloat16* __restrict__ weight,
                                                      const __nv_bfloat16* __restrict__ bias, float eps,
                                                      __nv_bfloat16* __restrict__ out, float* __restrict__ save_invstd,
                                                      uint32_t nvec, uint32_t groups, uint32_t active, uint32_t channels) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (blockIdx.x == 0)
    for (uint32_t c = threadIdx.x; c < channels; c += blockDim.x) save_invstd[c] = rsqrtf(var[c] + eps);
  if (t >= active) return;
  const uint32_t c0 = (t % groups) * 8;
  float m[8], is[8], w[8], b[8];
  {
    const float4 m0 = __ldg(reinterpret_cast<const float4*>(mean + c0)), m1 = __ldg(reinterpret_cast<const float4*>(mean + c0 + 4));
    const float4 v0 = __ldg(reinterpret_cast<const float4*>(var + c0)), v1 = __ldg(reinterpret_cast<const float4*>(var + c0 + 4));
    m[0] = m0.x; m[1] = m0.y; m[2] = m0.z; m[3] = m0.w; m[4] = m1.x; m[5] = m1.y; m[6] = m1.z; m[7] = m1.w;
    is[0] = v0.x; is[1] = v0.y; is[2] = v0.z; is[3] = v0.w; is[4] = v1.x; is[5] = v1.y; is[6] = v1.z; is[7] = v1.w;
#pragma unroll
    for (int j = 0; j < 8; ++j) is[j] = rsqrtf(is[j] + eps);
    unpack16<STK_BF16>(__ldg(reinterpret_cast<const uint4*>(weight + c0)), w);
    unpack16<STK_BF16>(__ldg(reinterpret_cast<const uint4*>(bias + c0)), b);
  }
  const uint4* xv = reinterpret_cast<const uint4*>(x);
  const uint4* rv = reinterpret_cast<const uint4*>(r);
  uint4* ov = reinterpret_cast<uint4*>(out);
  for (uint32_t v = t; v < nvec; v += active) {
    float xf[8], rf[8];
    unpack16<STK_BF16>(__ldg(xv + v), xf);
    if (kResidual) unpack16<STK_BF16>(__ldg(rv + v), rf);
    uint16_t o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      uint16_t z = bf16_bits(w[j] * (xf[j] - m[j]) * is[j] + b[j]);
      if (kResidual) z = bf16_bits(bf16_val(z) + rf[j]);
      const float zf = bf16_val(z);
      o[j] = isnan(zf) ? z : bf16_bits(fmaxf(zf, 0.f));
    }
    ov[v] = make_uint4(o[0] | uint32_t(o[1]) << 16, o[2] | uint32_t(o[3]) << 16, o[4] | uint32_t(o[5]) << 16,
                       o[6] | uint32_t(o[7]) << 16);
  }
}

}  // namespace stk

using namespace stk;

extern "C" {

int stk_bn_act(stk_ctx* c, const void* x, const void* residual, const float* mean, const float* var, const void* weight,
               const void* bias, double eps, void* out, float* save_invstd, size_t numel, size_t channels, void* stream) {
  STK_REQUIRE(c, c && x && mean && var && weight && bias && out && save_invstd, "stk_bn_act: NULL argument");
  STK_REQUIRE(c, channels > 0 && channels % 8 == 0 && numel % channels == 0, "stk_bn_act: channels must be a positive multiple of 8 dividing numel");
  STK_REQUIRE(c, numel < (size_t(1) << 31), "stk_bn_act: numel must be below 2^31");
  const uintptr_t align = uintptr_t(x) | uintptr_t(residual) | uintptr_t(mean) | uintptr_t(var) | uintptr_t(weight) |
                          uintptr_t(bias) | uintptr_t(out);
  STK_REQUIRE(c, align % 16 == 0, "stk_bn_act: every tensor must be 16-byte aligned");
  DeviceGuard g(c->device);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const uint32_t nvec = uint32_t(numel / 8), groups = uint32_t(channels / 8);
  auto kern = residual ? k_bn_act<true> : k_bn_act<false>;
  const size_t resident = size_t(blocks_per_sm(c, kern, kBnThreads)) * c->sm_count;
  // enough threads to cover every channel group once, at most one resident wave, at most one thread per vector
  size_t blocks = std::min(resident, (size_t(nvec) + kBnThreads - 1) / kBnThreads);
  blocks = std::max(blocks, (size_t(groups) + kBnThreads - 1) / kBnThreads);
  const uint32_t active = uint32_t(blocks * kBnThreads / groups * groups);
  kern<<<unsigned(blocks), kBnThreads, 0, s>>>(static_cast<const __nv_bfloat16*>(x), static_cast<const __nv_bfloat16*>(residual),
                                               mean, var, static_cast<const __nv_bfloat16*>(weight),
                                               static_cast<const __nv_bfloat16*>(bias), float(eps),
                                               static_cast<__nv_bfloat16*>(out), save_invstd, nvec, groups, active,
                                               uint32_t(channels));
  STK_CUDA(c, cudaGetLastError());
  return STK_OK;
}

}  // extern "C"
