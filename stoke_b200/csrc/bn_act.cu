// bn_act.cu -- BatchNorm apply (+ residual add) + activation in one pass over a bf16 NHWC activation, for training-mode
// BatchNorm whose statistics torch has already reduced (stk_bn_act_ex in include/stoke_b200.h), and its backward.
//
// Purely elementwise.  Every rounding of the unfused torch sequence is kept, so the result is bit-identical to it:
//   y = bf16(w * (x - mean) * invstd + b)        batch_norm_transform_input_channels_last_kernel (FADD, FMUL, FFMA)
//   z = bf16(float(y) + float(r))                `out += identity` on bf16 (fp32 add, one rounding; ReLU only)
//   out = act(z)                                 torch's CUDA activation kernel on a bf16 input (act_out below)
//   invstd = rsqrtf(var + eps)                   batch_norm_update_stats_and_invert
// Bytes per element: x read 2 + out write 2 (+ residual read 2).  The unfused chain moves 8 (15 with the residual).
#include <algorithm>
#include <cuda/atomic>

#include "common.cuh"
#include "ctx.cuh"

namespace stk {

constexpr int kBnThreads = 256;

__device__ __forceinline__ uint16_t bf16_bits(float f) { return __bfloat16_as_ushort(__float2bfloat16_rn(f)); }
__device__ __forceinline__ float bf16_val(uint16_t u) { return __uint_as_float(uint32_t(u) << 16); }

// The BatchNorm apply y = bf16(w * (x - mean) * invstd + b), as torch's channels-last transform kernel rounds it.  The
// forward activates it and the backward recomputes the activation's input from it, so the two cannot disagree.
__device__ __forceinline__ uint16_t bn_apply(float x, float m, float is, float w, float b) {
  return bf16_bits(__fmaf_rn(__fmul_rn(w, __fsub_rn(x, m)), is, b));
}

// The activation of a bf16 value z, as torch 2.11's CUDA kernel evaluates it: in fp32 (opmath) with one rounding, IEEE
// division and libdevice expf (the library is built without --use_fast_math, as torch is).
//   ReLU       relu_ = clamp_min_(0): a NaN keeps its bits
//   SiLU       x / (1 + exp(-x))
//   Hardswish  x * min(max(x + 3, 0), 6) * (1/6)   (std::min / std::max; a NaN gives NaN either way)
//   ReLU6      hardtanh = clamp(x, 0, 6): a NaN keeps its bits, otherwise fminf(fmaxf(x, 0), 6)
template <int kAct>
__device__ __forceinline__ uint16_t act_out(uint16_t z) {
  const float f = bf16_val(z);
  if (kAct == STK_ACT_RELU) return isnan(f) ? z : bf16_bits(fmaxf(f, 0.f));
  if (kAct == STK_ACT_SILU) return bf16_bits(__fdiv_rn(f, __fadd_rn(1.f, expf(-f))));
  if (kAct == STK_ACT_HARDSWISH) {
    float t = __fadd_rn(f, 3.f);
    t = t < 0.f ? 0.f : t;
    t = 6.f < t ? 6.f : t;
    return bf16_bits(__fmul_rn(__fmul_rn(f, t), 1.0f / 6.0f));
  }
  return isnan(f) ? z : bf16_bits(fminf(fmaxf(f, 0.f), 6.f));
}

// The activation's backward at input y (a bf16 value) for incoming gradient d, in fp32 before torch's rounding to bf16:
//   SiLU       silu_backward: s = 1 / (1 + exp(-y)); d * s * (1 + y * (1 - s)), the last product-sum contracted (FFMA)
//   Hardswish  hardswish_backward: y <= -3 ? 0 : y < 3 ? d * (y / 3 + 0.5) : d
//   ReLU6      hardtanh_backward(d, y, 0, 6): y <= 0 || y >= 6 ? 0 : d
// (ReLU's threshold_backward keeps the gradient's bits instead; it is mask_grad below.)
template <int kAct>
__device__ __forceinline__ float act_grad(float d, float y) {
  if (kAct == STK_ACT_SILU) {
    const float s = __fdiv_rn(1.f, __fadd_rn(1.f, expf(-y)));
    return __fmul_rn(__fmul_rn(d, s), __fmaf_rn(y, __fsub_rn(1.f, s), 1.f));
  }
  if (kAct == STK_ACT_HARDSWISH) return y <= -3.f ? 0.f : y < 3.f ? __fmul_rn(d, __fadd_rn(__fdiv_rn(y, 3.f), 0.5f)) : d;
  return y <= 0.f || y >= 6.f ? 0.f : d;
}

__device__ __forceinline__ uint4 pack8(const uint16_t (&o)[8]) {
  return make_uint4(o[0] | uint32_t(o[1]) << 16, o[2] | uint32_t(o[3]) << 16, o[4] | uint32_t(o[5]) << 16,
                    o[6] | uint32_t(o[7]) << 16);
}

// The apply over the vectors v = t, t + active, ... of one channel group, whose parameters the caller loaded.
template <int kAct, bool kResidual>
__device__ __forceinline__ void bn_act_vectors(const uint4* __restrict__ xv, const uint4* __restrict__ rv, uint4* __restrict__ ov,
                                               const float (&m)[8], const float (&is)[8], const float (&w)[8],
                                               const float (&b)[8], uint32_t t, uint32_t nvec, uint32_t active) {
  for (uint32_t v = t; v < nvec; v += active) {
    float xf[8], rf[8];
    unpack16<STK_BF16>(__ldg(xv + v), xf);
    if (kResidual) unpack16<STK_BF16>(__ldg(rv + v), rf);
    uint16_t o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      uint16_t z = bn_apply(xf[j], m[j], is[j], w[j], b[j]);
      if (kResidual) z = bf16_bits(bf16_val(z) + rf[j]);
      o[j] = act_out<kAct>(z);
    }
    ov[v] = pack8(o);
  }
}

// Thread t owns channel group t % G (G = C / 8) and walks rows t / G, t / G + T / G, ...: T (the active thread count) is a
// multiple of G, so the per-channel parameters stay in registers for the whole loop.
template <int kAct, bool kResidual>
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
  bn_act_vectors<kAct, kResidual>(reinterpret_cast<const uint4*>(x), reinterpret_cast<const uint4*>(r),
                                  reinterpret_cast<uint4*>(out), m, is, w, b, t, nvec, active);
}

// ---- backward ------------------------------------------------------------------------------------------------------
// The activation's backward g (ReLU's threshold_backward g = !(out <= 0) ? grad : +0, or act_grad) is folded into the
// two passes of torch's channels-last BatchNorm backward (batch_norm_backward_reduce_channels_last_kernel,
// batch_norm_backward_elemt_channels_last_kernel), whose sums are reproduced in torch's order, so every result is
// bit-identical to the unfused chain.  The ReLU mask comes from out at sites with a residual (where g is also written:
// it is the residual's gradient); every other site recomputes y = bn_apply(x) (relu(y) <= 0 exactly when y <= 0).
// Bytes per element: 4 + 6 without the residual, 8 + 6 with it; the unfused chain moves 16.
constexpr int kBwdThreads = 256;
constexpr int kChains = 4;   // torch's ELEMENTS_PER_ITER: accumulators per virtual thread

// 16-byte vector of 8 bf16 grads with the elements whose mask is off replaced by +0 (bits kept, NaN payloads included)
__device__ __forceinline__ uint4 mask_grad(const uint4& g, const bool (&pass)[8]) {
  const uint32_t m[4] = {(pass[0] ? 0xffffu : 0u) | (pass[1] ? 0xffff0000u : 0u), (pass[2] ? 0xffffu : 0u) | (pass[3] ? 0xffff0000u : 0u),
                         (pass[4] ? 0xffffu : 0u) | (pass[5] ? 0xffff0000u : 0u), (pass[6] ? 0xffffu : 0u) | (pass[7] ? 0xffff0000u : 0u)};
  return make_uint4(g.x & m[0], g.y & m[1], g.z & m[2], g.w & m[3]);
}

// g at a site without a residual, from the activation's input y = bn_apply(x) recomputed per element
template <int kAct>
__device__ __forceinline__ uint4 act_backward8(const uint4& gv, const float (&xf)[8], const float (&m)[8], const float (&is)[8],
                                               const float (&w)[8], const float (&b)[8]) {
  if (kAct == STK_ACT_RELU) {
    bool pass[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) pass[k] = !(bf16_val(bn_apply(xf[k], m[k], is[k], w[k], b[k])) <= 0.f);
    return mask_grad(gv, pass);
  }
  float d[8];
  unpack16<STK_BF16>(gv, d);
  uint16_t o[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) o[k] = bf16_bits(act_grad<kAct>(d[k], bf16_val(bn_apply(xf[k], m[k], is[k], w[k], b[k]))));
  return pack8(o);
}

__device__ __forceinline__ void load8(const float* __restrict__ p, float (&f)[8]) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p + 4));
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}

// sum_dy = sum g and sum_dy_xmu = sum g * (x - mean) per channel, in torch's order.  torch runs a (block_x, block_y) x
// (grid_x, grid_y) grid; for one channel, virtual thread (ty, by) keeps kChains accumulators, chain j adding rows
// m0 + (kChains * i + j) * S, i < loops (S = block_y * grid_y, m0 = by * block_y + ty; rows past the end add g = x = 0),
// as acc += g and acc = fma(g, x - mean, acc).  The chains are folded 0 += 1, 2, 3, then halved over ty (offsets
// block_y / 2 .. 1).  Here one real thread runs one chain of one virtual thread for 8 channels; a block holds every ty
// of its by for kBwdThreads / (kChains * block_y) channel groups.  With grid_y == 1 the block's sums are final;
// otherwise they go to the workspace partials and k_bn_bwd_finish adds them.  g_out receives g: the residual's gradient
// (ReLU), or the optional grad_pre of another activation.  ReLU without a residual has no g_out: a run-time checked
// store there would take its instantiation from 80 to 99 registers.  kSum (residual sites): the output's gradient
// arrives in two parts, grad and grad2, summed first as autograd's bf16 add sums them: bf16(float(grad) + float(grad2)).
// kTwo (residual sites whose residual is a second BatchNorm's output, relu(bn(x) + bn2(x2))): torch's backward of bn2
// sees the same g on the same grid, so sum_dy serves both; a third row sums g * (x2 - mean2) in the same order.
struct BnBwdSecond {   // the second BatchNorm of a kTwo site
  const uint4* x;
  const float* mean;
  const float* invstd;
  const __nv_bfloat16* weight;
  float* ws;           // its sum_dy_xmu [C], then per-block partials [grid_y][C]
  __nv_bfloat16* dweight;
  __nv_bfloat16* dbias;
  uint4* dx;
};

template <int kAct, bool kResidual, bool kSum = false, bool kTwo = false>
__global__ void __launch_bounds__(kBwdThreads) k_bn_bwd_reduce(const uint4* __restrict__ grad, const uint4* __restrict__ grad2,
                                                               const uint4* __restrict__ x,
                                                               const uint4* __restrict__ out, const float* __restrict__ mean,
                                                               const float* __restrict__ invstd,
                                                               const __nv_bfloat16* __restrict__ weight,
                                                               const __nv_bfloat16* __restrict__ bias, uint4* __restrict__ g_out,
                                                               float* __restrict__ ws, __nv_bfloat16* __restrict__ dweight,
                                                               __nv_bfloat16* __restrict__ dbias, uint32_t rows,
                                                               uint32_t groups, uint32_t block_y, uint32_t loops,
                                                               const BnBwdSecond s2) {
  constexpr int kS = kTwo ? 24 : 16;   // sums per thread
  // per thread: 8 sums of g, then 8 sums of g * (x - mean) (then 8 of g * (x2 - mean2))
  __shared__ float4 sh[kBwdThreads][kS / 4];
  const uint32_t t = threadIdx.x, gb = kBwdThreads / (kChains * block_y);
  const uint32_t cgl = t % gb, j = t / gb % kChains, ty = t / (gb * kChains);
  const uint32_t cg = blockIdx.x * gb + cgl, c0 = cg * 8, channels = groups * 8;
  const bool live = cg < groups;
  float sdy[8], sxm[8], sxm2[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) sdy[k] = sxm[k] = sxm2[k] = 0.f;
  if (live) {
    float m[8], is[8], w[8], b[8], m2[8];
    if (!kResidual) {
      load8(invstd + c0, is);
      unpack16<STK_BF16>(__ldg(reinterpret_cast<const uint4*>(weight + c0)), w);
      unpack16<STK_BF16>(__ldg(reinterpret_cast<const uint4*>(bias + c0)), b);
    }
    load8(mean + c0, m);
    if (kTwo) load8(s2.mean + c0, m2);
    const uint32_t stride = block_y * gridDim.y, m0 = blockIdx.y * block_y + ty;
#pragma unroll 2
    for (uint32_t i = 0; i < loops; ++i) {
      const uint32_t row = m0 + (kChains * i + j) * stride;
      const bool in = row < rows;
      const size_t v = size_t(row) * groups + cg;
      const uint4 zero = make_uint4(0, 0, 0, 0);
      uint4 gv = in ? __ldg(grad + v) : zero;
      const uint4 xv = in ? __ldg(x + v) : zero;
      float xf[8], gf[8], mf[8];
      if (kSum) {
        float g2[8];
        unpack16<STK_BF16>(gv, gf);
        unpack16<STK_BF16>(in ? __ldg(grad2 + v) : zero, g2);
        uint16_t o[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) o[k] = bf16_bits(__fadd_rn(gf[k], g2[k]));
        gv = pack8(o);
      }
      unpack16<STK_BF16>(xv, xf);
      uint4 g;
      if (kResidual) {
        bool pass[8];
        unpack16<STK_BF16>(in ? __ldg(out + v) : zero, mf);
#pragma unroll
        for (int k = 0; k < 8; ++k) pass[k] = !(mf[k] <= 0.f);
        g = mask_grad(gv, pass);
      } else if (kAct == STK_ACT_RELU || in) {
        g = act_backward8<kAct>(gv, xf, m, is, w, b);
      } else {
        // a row past the end adds g = +0 as in torch, whose activation backward never sees it: SiLU's backward of a
        // zero gradient is NaN where bn_apply(0) overflows to +-inf (0 * s * fma(inf, 1 - s, 1))
        g = zero;
      }
      if ((kResidual || (kAct != STK_ACT_RELU && g_out != nullptr)) && in) g_out[v] = g;
      unpack16<STK_BF16>(g, gf);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        sdy[k] = __fadd_rn(sdy[k], gf[k]);
        sxm[k] = __fmaf_rn(gf[k], __fsub_rn(xf[k], m[k]), sxm[k]);
      }
      if (kTwo) {
        unpack16<STK_BF16>(in ? __ldg(s2.x + v) : zero, xf);
#pragma unroll
        for (int k = 0; k < 8; ++k) sxm2[k] = __fmaf_rn(gf[k], __fsub_rn(xf[k], m2[k]), sxm2[k]);
      }
    }
  }
  sh[t][0] = make_float4(sdy[0], sdy[1], sdy[2], sdy[3]);
  sh[t][1] = make_float4(sdy[4], sdy[5], sdy[6], sdy[7]);
  sh[t][2] = make_float4(sxm[0], sxm[1], sxm[2], sxm[3]);
  sh[t][3] = make_float4(sxm[4], sxm[5], sxm[6], sxm[7]);
  if (kTwo) {
    sh[t][kS / 4 - 2] = make_float4(sxm2[0], sxm2[1], sxm2[2], sxm2[3]);
    sh[t][kS / 4 - 1] = make_float4(sxm2[4], sxm2[5], sxm2[6], sxm2[7]);
  }
  __syncthreads();
  // fold the chains, then halve over ty; thread (cgl, ty) of chain 0 owns the slot of that virtual thread
  const bool owner = j == 0;
  float s[kS];
  if (owner) {
    const float* p = reinterpret_cast<const float*>(sh[t]);
#pragma unroll
    for (int k = 0; k < kS; ++k) s[k] = p[k];
#pragma unroll
    for (int q = 1; q < kChains; ++q) {
      const float* r = reinterpret_cast<const float*>(sh[t + q * gb]);
#pragma unroll
      for (int k = 0; k < kS; ++k) s[k] = __fadd_rn(s[k], r[k]);
    }
  }
  __syncthreads();
  for (uint32_t off = block_y / 2; off > 0; off >>= 1) {
    if (owner && ty < 2 * off) {
      float* p = reinterpret_cast<float*>(sh[t]);
#pragma unroll
      for (int k = 0; k < kS; ++k) p[k] = s[k];
    }
    __syncthreads();
    if (owner && ty < off) {
      const float* r = reinterpret_cast<const float*>(sh[t + off * gb * kChains]);
#pragma unroll
      for (int k = 0; k < kS; ++k) s[k] = __fadd_rn(s[k], r[k]);
    }
    __syncthreads();
  }
  if (!(owner && ty == 0 && live)) return;
  if (kTwo) {
    if (gridDim.y == 1) {
      float is2[8];
      load8(s2.invstd + c0, is2);
      uint16_t dw[8], db[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        s2.ws[c0 + k] = s[16 + k];
        db[k] = bf16_bits(s[k]);
        dw[k] = bf16_bits(__fmul_rn(s[16 + k], is2[k]));
      }
      *reinterpret_cast<uint4*>(s2.dbias + c0) = pack8(db);
      *reinterpret_cast<uint4*>(s2.dweight + c0) = pack8(dw);
    } else {
      float* p = s2.ws + channels + size_t(blockIdx.y) * channels + c0;
#pragma unroll
      for (int k = 0; k < 8; ++k) p[k] = s[16 + k];
    }
  }
  if (gridDim.y == 1) {
    float is[8];
    load8(invstd + c0, is);
    uint16_t dw[8], db[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      ws[c0 + k] = s[k];
      ws[channels + c0 + k] = s[8 + k];
      db[k] = bf16_bits(s[k]);
      dw[k] = bf16_bits(__fmul_rn(s[8 + k], is[k]));
    }
    *reinterpret_cast<uint4*>(dbias + c0) = make_uint4(db[0] | uint32_t(db[1]) << 16, db[2] | uint32_t(db[3]) << 16,
                                                       db[4] | uint32_t(db[5]) << 16, db[6] | uint32_t(db[7]) << 16);
    *reinterpret_cast<uint4*>(dweight + c0) = make_uint4(dw[0] | uint32_t(dw[1]) << 16, dw[2] | uint32_t(dw[3]) << 16,
                                                         dw[4] | uint32_t(dw[5]) << 16, dw[6] | uint32_t(dw[7]) << 16);
  } else {
    float* pdy = ws + 2 * channels + size_t(blockIdx.y) * channels + c0;
    float* pxm = pdy + size_t(gridDim.y) * channels;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      pdy[k] = s[k];
      pxm[k] = s[8 + k];
    }
  }
}

// torch's cross-block finish: thread ty adds the partials of blocks ty, ty + block_y, ... from +0, then the halving
// tree over ty.  One thread per (channel, ty).  kTwo: the third row too (the second BatchNorm's sum_dy_xmu).
template <bool kTwo>
__global__ void __launch_bounds__(kBwdThreads) k_bn_bwd_finish(float* __restrict__ ws, const float* __restrict__ invstd,
                                                               __nv_bfloat16* __restrict__ dweight,
                                                               __nv_bfloat16* __restrict__ dbias, uint32_t channels,
                                                               uint32_t block_y, uint32_t grid_y, const BnBwdSecond s2) {
  __shared__ float sh[kTwo ? 3 : 2][kBwdThreads];
  const uint32_t t = threadIdx.x, cb = kBwdThreads / block_y, ty = t / cb, c = blockIdx.x * cb + t % cb;
  const bool live = c < channels;
  const float* pdy = ws + 2 * channels;
  const float* pxm = pdy + size_t(grid_y) * channels;
  const float* pxm2 = s2.ws + channels;
  float dy = 0.f, xm = 0.f, xm2 = 0.f;
  if (live)
    for (uint32_t y = ty; y < grid_y; y += block_y) {
      dy = __fadd_rn(dy, pdy[size_t(y) * channels + c]);
      xm = __fadd_rn(xm, pxm[size_t(y) * channels + c]);
      if (kTwo) xm2 = __fadd_rn(xm2, pxm2[size_t(y) * channels + c]);
    }
  for (uint32_t off = block_y / 2; off > 0; off >>= 1) {
    sh[0][t] = dy;
    sh[1][t] = xm;
    if (kTwo) sh[kTwo ? 2 : 0][t] = xm2;
    __syncthreads();
    if (ty < off) {
      dy = __fadd_rn(dy, sh[0][t + off * cb]);
      xm = __fadd_rn(xm, sh[1][t + off * cb]);
      if (kTwo) xm2 = __fadd_rn(xm2, sh[kTwo ? 2 : 0][t + off * cb]);
    }
    __syncthreads();
  }
  if (ty != 0 || !live) return;
  ws[c] = dy;
  ws[channels + c] = xm;
  dbias[c] = __float2bfloat16_rn(dy);
  dweight[c] = __float2bfloat16_rn(__fmul_rn(xm, invstd[c]));
  if (kTwo) {
    s2.ws[c] = xm2;
    s2.dbias[c] = __float2bfloat16_rn(dy);
    s2.dweight[c] = __float2bfloat16_rn(__fmul_rn(xm2, s2.invstd[c]));
  }
}

// dx = bf16(((g - sum_dy * n) - (x - mean) * k1) * k2), k1 = invstd * invstd * sum_dy_xmu * n, k2 = w * invstd,
// n = float(1.0 / rows): torch's channels-last elementwise backward, whose SASS contracts both subtractions with their
// products (FFMA -sum_dy * n + g; FADD x - mean; FFMA -k1 * (x - mean) + t; FMUL k2).  Thread layout as in k_bn_act.
// kTwo: the second BatchNorm's dx2 from the same g and sum_dy, with its own mean, k1 and k2.
template <int kAct, bool kResidual, bool kTwo = false>
__global__ void __launch_bounds__(kBnThreads) k_bn_bwd_elemt(const uint4* __restrict__ grad, const uint4* __restrict__ x,
                                                            const float* __restrict__ mean, const float* __restrict__ invstd,
                                                            const __nv_bfloat16* __restrict__ weight,
                                                            const __nv_bfloat16* __restrict__ bias,
                                                            const float* __restrict__ ws, uint4* __restrict__ dx, float n,
                                                            uint32_t nvec, uint32_t groups, uint32_t active,
                                                            const BnBwdSecond s2) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= active) return;
  const uint32_t c0 = (t % groups) * 8, channels = groups * 8;
  if (kTwo) {
    float m[8], m2[8], sdy[8], k1[8], k2[8], k1b[8], k2b[8];
    {
      float is[8], w[8], sxm[8];
      load8(mean + c0, m);
      load8(invstd + c0, is);
      load8(ws + c0, sdy);
      load8(ws + channels + c0, sxm);
      unpack16<STK_BF16>(__ldg(reinterpret_cast<const uint4*>(weight + c0)), w);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        k1[k] = __fmul_rn(__fmul_rn(__fmul_rn(is[k], is[k]), sxm[k]), n);
        k2[k] = __fmul_rn(w[k], is[k]);
      }
      load8(s2.mean + c0, m2);
      load8(s2.invstd + c0, is);
      load8(s2.ws + c0, sxm);
      unpack16<STK_BF16>(__ldg(reinterpret_cast<const uint4*>(s2.weight + c0)), w);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        k1b[k] = __fmul_rn(__fmul_rn(__fmul_rn(is[k], is[k]), sxm[k]), n);
        k2b[k] = __fmul_rn(w[k], is[k]);
      }
    }
    for (uint32_t v = t; v < nvec; v += active) {
      float xf[8], x2f[8], gf[8];
      unpack16<STK_BF16>(__ldg(x + v), xf);
      unpack16<STK_BF16>(__ldg(s2.x + v), x2f);
      unpack16<STK_BF16>(__ldg(grad + v), gf);
      uint16_t o[8], o2[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float gc = __fmaf_rn(-sdy[k], n, gf[k]);
        o[k] = bf16_bits(__fmul_rn(__fmaf_rn(-__fsub_rn(xf[k], m[k]), k1[k], gc), k2[k]));
        o2[k] = bf16_bits(__fmul_rn(__fmaf_rn(-__fsub_rn(x2f[k], m2[k]), k1b[k], gc), k2b[k]));
      }
      dx[v] = pack8(o);
      s2.dx[v] = pack8(o2);
    }
    return;
  }
  float m[8], is[8], w[8], b[8], sdy[8], k1[8], k2[8];
  {
    float sxm[8];
    load8(mean + c0, m);
    load8(invstd + c0, is);
    load8(ws + c0, sdy);
    load8(ws + channels + c0, sxm);
    unpack16<STK_BF16>(__ldg(reinterpret_cast<const uint4*>(weight + c0)), w);
    if (!kResidual) unpack16<STK_BF16>(__ldg(reinterpret_cast<const uint4*>(bias + c0)), b);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      k1[k] = __fmul_rn(__fmul_rn(__fmul_rn(is[k], is[k]), sxm[k]), n);
      k2[k] = __fmul_rn(w[k], is[k]);
    }
  }
  for (uint32_t v = t; v < nvec; v += active) {
    float xf[8], gf[8];
    unpack16<STK_BF16>(__ldg(x + v), xf);
    uint4 g = __ldg(grad + v);
    if (!kResidual) g = act_backward8<kAct>(g, xf, m, is, w, b);
    unpack16<STK_BF16>(g, gf);
    uint16_t o[8];
#pragma unroll
    for (int k = 0; k < 8; ++k)
      o[k] = bf16_bits(__fmul_rn(__fmaf_rn(-__fsub_rn(xf[k], m[k]), k1[k], __fmaf_rn(-sdy[k], n, gf[k])), k2[k]));
    dx[v] = make_uint4(o[0] | uint32_t(o[1]) << 16, o[2] | uint32_t(o[3]) << 16, o[4] | uint32_t(o[5]) << 16,
                       o[6] | uint32_t(o[7]) << 16);
  }
}

// torch's flexible_launch_configs(rows, channels, coop = true) with MAX_BLOCK_SIZE 512, as the channels-last backward
// reduce launches it: the only inputs of its summation order besides the row count.
struct BnBwdConfig {
  uint32_t block_y, grid_y, loops;
};

static uint32_t last_pow2(uint32_t n) {
  uint32_t p = 1;
  while (p <= n / 2) p *= 2;
  return p;
}

static BnBwdConfig bn_bwd_config(uint32_t rows, uint32_t channels) {
  const uint32_t block_x = std::min(last_pow2(channels), 32u);
  const uint32_t block_y = std::min(last_pow2((rows + 15) / 16), 512u / block_x);
  uint32_t grid_y = std::min((rows + block_y * 16 - 1) / (block_y * 16), 128u);
  if (grid_y < 8) grid_y = 1;
  return {block_y, grid_y, 1 + (rows - 1) / (block_y * grid_y * kChains)};
}

// ---- forward with the statistics -----------------------------------------------------------------------------------
// k_bn_stats_act: torch.batch_norm_update_stats followed by k_bn_act's apply in one cooperative launch of resident blocks,
// in three phases separated by grid barriers.  Bytes per element: x read twice (2 + 2; the second read hits L2 for the
// smaller sites) + out write 2 (+ residual read 2).  The unfused forward also launches a semaphore fill and the
// running-statistics update.
//  1. Welford partials in the order of torch's batch_norm_collect_statistics_channels_last_kernel<Var, BFloat16, float, 4>,
//     launched as flexible_launch_configs(R, C, coop) (the same (block_y, grid_y, loops) as the backward reduce).
//     Virtual thread (ty, by) keeps kChains chains; chain j takes rows m0 + (kChains * i + j) * S, i < loops, as
//       valid row:  n++, inv = 1 / float(n), d0 = x - mean, mean = fma(d0, inv, mean), d1 = x - mean, m2 = fma(d0 * d1, 1, m2)
//       past R:     the same with x = inv = 0 and 0 in place of 1 (so a -0 mean becomes +0, an infinite one NaN, as in torch)
//     then folds chains 1..3 into chain 0 and halves over ty (welford_merge).  Real threads map as in k_bn_bwd_reduce;
//     a persistent grid walks the (channel block, by) work items.  With grid_y == 1 the block's result is final.
//  2. torch's last-block merge: thread ty merges the partials of blocks ty, ty + block_y, ... from (0, 0, 0), then the
//     halving tree.  The channel's owner writes save_mean, save_invstd = rsqrtf(m2 / n + eps) (k_bn_act's formula) and
//     the running statistics as torch's batch_norm_update_stats kernel computes them in float:
//       running = fma(stat, momentum, (1 - momentum) * running),  stat = mean, or var * float(R / (R - 1.0)) for the var
//  3. k_bn_act's apply from save_mean / save_invstd.
struct BnStatsArgs {
  const uint4* x;
  const uint4* r;
  const __nv_bfloat16* weight;
  const __nv_bfloat16* bias;
  void* running_mean;
  void* running_var;
  uint4* out;
  float* save_mean;
  float* save_invstd;
  float* ws;          // [grid_y][C] partial means, then m2s, then counts (int); the second BatchNorm's after them
  uint32_t* bar;      // grid barrier: arrival count, generation
  float eps, momentum, one_minus_momentum, bessel;
  uint32_t rows, groups, block_y, grid_y, loops, nvec, active;
  // the residual's BatchNorm at a kTwo site (its input is r)
  const __nv_bfloat16* weight2;
  const __nv_bfloat16* bias2;
  void* running_mean2;
  void* running_var2;
  float* save_mean2;
  float* save_invstd2;
  float eps2, momentum2, one_minus_momentum2;
};

// A barrier over the whole (co-resident) grid.  The arrival count returns to 0 at every barrier and the generation only
// grows, so the words need no reset between launches.
__device__ __forceinline__ void grid_barrier(uint32_t* bar) {
  __syncthreads();
  if (threadIdx.x == 0) {
    cuda::atomic_ref<uint32_t, cuda::thread_scope_device> arrived(bar[0]), gen(bar[1]);
    const uint32_t g = gen.load(cuda::memory_order_relaxed);
    __threadfence();
    if (arrived.fetch_add(1, cuda::memory_order_acq_rel) == gridDim.x - 1) {
      arrived.store(0, cuda::memory_order_relaxed);
      gen.store(g + 1, cuda::memory_order_release);
    } else {
      while (gen.load(cuda::memory_order_acquire) == g) __nanosleep(32);
    }
    __threadfence();
  }
  __syncthreads();
}

// torch's welford_merge_element for 8 channels of one count: (n, mean, m2) += (n2, mean2, m22), factor = 1 / float(max(1,
// n + n2)), m2 += m22 + d * d * n2 * n * factor (the last product contracted with m22), mean = (mean2 * n2 + mean * n) *
// factor.  torch's SASS contracts that sum differently at its two call sites: fma(mean2, n2, mean * n) where a virtual
// thread folds its chains (kChainFold), fma(mean, n, mean2 * n2) in the vertical tree and the cross-block merge.
template <bool kChainFold, int K>
__device__ __forceinline__ void welford_merge(int& n, float (&mean)[K], float (&m2)[K], int n2, const float* mean2,
                                              const float* m22) {
  const float factor = __fdiv_rn(1.f, __int2float_rn(max(1, n + n2)));
  const float fn = __int2float_rn(n), fn2 = __int2float_rn(n2);
#pragma unroll
  for (int k = 0; k < K; ++k) {
    const float d = __fsub_rn(mean[k], mean2[k]);
    const float s = kChainFold ? __fmaf_rn(mean2[k], fn2, __fmul_rn(mean[k], fn)) : __fmaf_rn(mean[k], fn, __fmul_rn(mean2[k], fn2));
    m2[k] = __fadd_rn(__fmaf_rn(__fmul_rn(__fmul_rn(__fmul_rn(d, d), fn2), fn), factor, m22[k]), m2[k]);
    mean[k] = __fmul_rn(s, factor);
  }
  n += n2;
}

__device__ __forceinline__ float run_load(const float* p) { return *p; }
__device__ __forceinline__ float run_load(const __nv_bfloat16* p) { return __bfloat162float(*p); }
__device__ __forceinline__ void run_store(float* p, float v) { *p = v; }
__device__ __forceinline__ void run_store(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }

// the outputs of channel c from its final (mean, var = m2 / n), for BatchNorm `side` (1: the residual's at a kTwo site)
template <typename RunT>
__device__ __forceinline__ void bn_stats_finish(const BnStatsArgs& a, int side, uint32_t c, float mean, float var) {
  const float eps = side ? a.eps2 : a.eps, mom = side ? a.momentum2 : a.momentum;
  const float omm = side ? a.one_minus_momentum2 : a.one_minus_momentum;
  (side ? a.save_mean2 : a.save_mean)[c] = mean;
  (side ? a.save_invstd2 : a.save_invstd)[c] = rsqrtf(var + eps);
  RunT* rm = static_cast<RunT*>(side ? a.running_mean2 : a.running_mean) + c;
  RunT* rv = static_cast<RunT*>(side ? a.running_var2 : a.running_var) + c;
  run_store(rm, __fmaf_rn(mean, mom, __fmul_rn(omm, run_load(rm))));
  run_store(rv, __fmaf_rn(__fmul_rn(var, a.bessel), mom, __fmul_rn(omm, run_load(rv))));
}

// the halving tree over ty of torch's welford_merge_block_vertical; slot(t) is this thread's shared-memory slot, the
// partner's is slot + off * span.  Ends with the block synchronised.
template <int K>
__device__ __forceinline__ void welford_tree(bool owner, uint32_t ty, uint32_t block_y, uint32_t span, uint32_t slot, int& n,
                                             float (&mean)[K], float (&m2)[K], float (*shm)[2 * K], int* shn) {
  for (uint32_t off = block_y / 2; off > 0; off >>= 1) {
    if (owner && ty < 2 * off) {
#pragma unroll
      for (int k = 0; k < K; ++k) {
        shm[slot][k] = mean[k];
        shm[slot][K + k] = m2[k];
      }
      shn[slot] = n;
    }
    __syncthreads();
    if (owner && ty < off) {
      const uint32_t p = slot + off * span;
      welford_merge<false>(n, mean, m2, shn[p], shm[p], shm[p] + K);
    }
    __syncthreads();
  }
}

// kTwo (ReLU with a residual): the residual r is the input of a second BatchNorm (weight2, ...), whose statistics are
// gathered after x's in the same phases and applied before the add.
template <int kAct, bool kResidual, typename RunT, bool kTwo = false>
__global__ void __launch_bounds__(kBwdThreads, 3) k_bn_stats_act(const BnStatsArgs a) {
  __shared__ float shm[kBwdThreads][16];
  __shared__ int shn[kBwdThreads];
  const uint32_t t = threadIdx.x, channels = a.groups * 8;
  // phase 1
  {
    const uint32_t gb = kBwdThreads / (kChains * a.block_y);
    const uint32_t cgl = t % gb, j = t / gb % kChains, ty = t / (gb * kChains);
    const uint32_t nxb = (a.groups + gb - 1) / gb, stride = a.block_y * a.grid_y;
    // kTwo: x, then the residual through its own BatchNorm, one after the other (one Welford state at a time)
#pragma unroll 1
    for (int side = 0; side < (kTwo ? 2 : 1); ++side)
    for (uint32_t item = blockIdx.x; item < nxb * a.grid_y; item += gridDim.x) {
      const uint4* xs = side ? a.r : a.x;
      float* ws = a.ws + size_t(side) * 3 * a.grid_y * channels;
      const uint32_t by = item / nxb, cg = (item % nxb) * gb + cgl;
      const bool live = cg < a.groups;
      const uint32_t m0 = by * a.block_y + ty;
      int n = 0;
      float mean[8], m2[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) mean[k] = m2[k] = 0.f;
      // four rows' loads in flight before their (sequential) Welford updates
      for (uint32_t i0 = 0; i0 < a.loops; i0 += 4) {
        uint4 xv[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const uint32_t row = m0 + (kChains * (i0 + u) + j) * stride;
          xv[u] = live && i0 + u < a.loops && row < a.rows ? __ldg(xs + size_t(row) * a.groups + cg) : make_uint4(0, 0, 0, 0);
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          if (i0 + u >= a.loops) break;
          const bool in = live && m0 + (kChains * (i0 + u) + j) * stride < a.rows;
          float inv = 0.f, valid = 0.f;
          if (in) {
            ++n;
            inv = __fdiv_rn(1.f, __int2float_rn(n));
            valid = 1.f;
          }
          float xf[8];
          unpack16<STK_BF16>(xv[u], xf);
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            const float d0 = __fsub_rn(xf[k], mean[k]);
            mean[k] = __fmaf_rn(d0, inv, mean[k]);
            const float d1 = __fsub_rn(xf[k], mean[k]);
            m2[k] = __fmaf_rn(__fmul_rn(d0, d1), valid, m2[k]);
          }
        }
      }
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        shm[t][k] = mean[k];
        shm[t][8 + k] = m2[k];
      }
      shn[t] = n;
      __syncthreads();
      const bool owner = j == 0;
      if (owner)
        for (uint32_t q = 1; q < kChains; ++q) welford_merge<true>(n, mean, m2, shn[t + q * gb], shm[t + q * gb], shm[t + q * gb] + 8);
      __syncthreads();
      welford_tree(owner, ty, a.block_y, gb * kChains, t, n, mean, m2, shm, shn);
      if (owner && ty == 0 && live) {
        const uint32_t c0 = cg * 8;
        if (a.grid_y == 1) {
          for (int k = 0; k < 8; ++k) bn_stats_finish<RunT>(a, side, c0 + k, mean[k], __fdiv_rn(m2[k], __int2float_rn(n)));
        } else {
          float* pm = ws + size_t(by) * channels + c0;
          float* p2 = pm + size_t(a.grid_y) * channels;
          int* pn = reinterpret_cast<int*>(p2 + size_t(a.grid_y) * channels);
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            pm[k] = mean[k];
            p2[k] = m2[k];
            pn[k] = n;
          }
        }
      }
      __syncthreads();
    }
  }
  // phase 2
  if (a.grid_y > 1) {
    grid_barrier(a.bar);
    const uint32_t cb = kBwdThreads / a.block_y, ty = t / cb;
    float (*shm1)[2] = reinterpret_cast<float (*)[2]>(&shm[0][0]);
#pragma unroll 1
    for (int side = 0; side < (kTwo ? 2 : 1); ++side)
    for (uint32_t item = blockIdx.x; item * cb < channels; item += gridDim.x) {
      const float* pm = a.ws + size_t(side) * 3 * a.grid_y * channels;
      const float* p2 = pm + size_t(a.grid_y) * channels;
      const int* pn = reinterpret_cast<const int*>(p2 + size_t(a.grid_y) * channels);
      const uint32_t c = item * cb + t % cb;
      const bool live = c < channels;
      int n = 0;
      float mean[1] = {0.f}, m2[1] = {0.f};
      if (live)
        for (uint32_t y = ty; y < a.grid_y; y += a.block_y) {
          const size_t o = size_t(y) * channels + c;
          const float mn = __ldcg(pm + o), m2n = __ldcg(p2 + o);
          welford_merge<false>(n, mean, m2, __ldcg(pn + o), &mn, &m2n);
        }
      welford_tree(true, ty, a.block_y, cb, t, n, mean, m2, shm1, shn);
      if (ty == 0 && live) bn_stats_finish<RunT>(a, side, c, mean[0], __fdiv_rn(m2[0], __int2float_rn(n)));
    }
  }
  // phase 3
  grid_barrier(a.bar);
  const uint32_t tg = blockIdx.x * kBwdThreads + t;
  if (tg >= a.active) return;
  const uint32_t c0 = (tg % a.groups) * 8;
  float m[8], is[8], w[8], b[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    m[k] = __ldcg(a.save_mean + c0 + k);
    is[k] = __ldcg(a.save_invstd + c0 + k);
  }
  unpack16<STK_BF16>(__ldg(reinterpret_cast<const uint4*>(a.weight + c0)), w);
  unpack16<STK_BF16>(__ldg(reinterpret_cast<const uint4*>(a.bias + c0)), b);
  if (!kTwo) {
    bn_act_vectors<kAct, kResidual>(a.x, a.r, a.out, m, is, w, b, tg, a.nvec, a.active);
    return;
  }
  // z = bf16(float(bn_apply(x)) + float(bn_apply2(r))): `out += identity` with identity the residual BatchNorm's output
  float m2[8], is2[8], w2[8], b2[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    m2[k] = __ldcg(a.save_mean2 + c0 + k);
    is2[k] = __ldcg(a.save_invstd2 + c0 + k);
  }
  unpack16<STK_BF16>(__ldg(reinterpret_cast<const uint4*>(a.weight2 + c0)), w2);
  unpack16<STK_BF16>(__ldg(reinterpret_cast<const uint4*>(a.bias2 + c0)), b2);
  for (uint32_t v = tg; v < a.nvec; v += a.active) {
    float xf[8], rf[8];
    unpack16<STK_BF16>(__ldg(a.x + v), xf);
    unpack16<STK_BF16>(__ldg(a.r + v), rf);
    uint16_t o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint16_t y = bn_apply(xf[j], m[j], is[j], w[j], b[j]), y2 = bn_apply(rf[j], m2[j], is2[j], w2[j], b2[j]);
      o[j] = act_out<STK_ACT_RELU>(bf16_bits(bf16_val(y) + bf16_val(y2)));
    }
    a.out[v] = pack8(o);
  }
}

// k_bn_stats_act for one running-statistics dtype, in the form STK_BN_KERNEL takes
template <typename RunT>
struct BnStatsKernel {
  template <int kAct, bool kResidual>
  static constexpr auto k = k_bn_stats_act<kAct, kResidual, RunT>;
};

// The instantiation of `kernel` for (act, residual): every activation without a residual, and ReLU with one.
#define STK_BN_KERNEL(kernel, act, res)                                                                              \
  ((act) == STK_ACT_SILU        ? kernel<STK_ACT_SILU, false>                                                        \
   : (act) == STK_ACT_HARDSWISH ? kernel<STK_ACT_HARDSWISH, false>                                                   \
   : (act) == STK_ACT_RELU6     ? kernel<STK_ACT_RELU6, false>                                                       \
   : (res)                      ? kernel<STK_ACT_RELU, true>                                                         \
                                : kernel<STK_ACT_RELU, false>)

static bool act_valid(int act, bool residual) {
  return act >= STK_ACT_RELU && act <= STK_ACT_RELU6 && (act == STK_ACT_RELU || !residual);
}

}  // namespace stk

using namespace stk;

extern "C" {

int stk_bn_act_ex(stk_ctx* c, int act, const void* x, const void* residual, const float* mean, const float* var,
                  const void* weight, const void* bias, double eps, void* out, float* save_invstd, size_t numel,
                  size_t channels, void* stream) {
  STK_REQUIRE(c, c && x && mean && var && weight && bias && out && save_invstd, "stk_bn_act: NULL argument");
  STK_REQUIRE(c, act_valid(act, residual != nullptr),
              "stk_bn_act: act must be an STK_ACT_* kind, and only STK_ACT_RELU takes a residual");
  STK_REQUIRE(c, channels > 0 && channels % 8 == 0 && numel % channels == 0, "stk_bn_act: channels must be a positive multiple of 8 dividing numel");
  STK_REQUIRE(c, numel < (size_t(1) << 31), "stk_bn_act: numel must be below 2^31");
  const uintptr_t align = uintptr_t(x) | uintptr_t(residual) | uintptr_t(mean) | uintptr_t(var) | uintptr_t(weight) |
                          uintptr_t(bias) | uintptr_t(out);
  STK_REQUIRE(c, align % 16 == 0, "stk_bn_act: every tensor must be 16-byte aligned");
  DeviceGuard g(c->device);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const uint32_t nvec = uint32_t(numel / 8), groups = uint32_t(channels / 8);
  auto kern = STK_BN_KERNEL(k_bn_act, act, residual != nullptr);
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

int stk_bn_stats_act(stk_ctx* c, int act, const void* x, const void* residual, const void* weight, const void* bias,
                     void* running_mean, void* running_var, int running_dtype, double momentum, double eps, void* out,
                     float* save_mean, float* save_invstd, float* workspace, size_t numel, size_t channels, void* stream,
                     const void* weight2, const void* bias2, void* running_mean2, void* running_var2, double momentum2,
                     double eps2, float* save_mean2, float* save_invstd2) {
  STK_REQUIRE(c, c && x && weight && bias && running_mean && running_var && out && save_mean && save_invstd && workspace,
              "stk_bn_stats_act: NULL argument");
  STK_REQUIRE(c, act_valid(act, residual != nullptr),
              "stk_bn_stats_act: act must be an STK_ACT_* kind, and only STK_ACT_RELU takes a residual");
  const bool two = weight2 != nullptr;
  STK_REQUIRE(c, !two || (residual && bias2 && running_mean2 && running_var2 && save_mean2 && save_invstd2),
              "stk_bn_stats_act: a second BatchNorm needs a residual, bias2, running statistics and save_mean2 / save_invstd2");
  STK_REQUIRE(c, ((uintptr_t(weight2) | uintptr_t(bias2)) % 16) == 0, "stk_bn_stats_act: weight2 and bias2 must be 16-byte aligned");
  STK_REQUIRE(c, running_dtype == STK_F32 || running_dtype == STK_BF16, "stk_bn_stats_act: running statistics must be STK_F32 or STK_BF16");
  STK_REQUIRE(c, channels > 0 && channels % 8 == 0 && numel % channels == 0 && numel >= 2 * channels,
              "stk_bn_stats_act: channels must be a positive multiple of 8 dividing numel, with at least 2 rows");
  STK_REQUIRE(c, numel < (size_t(1) << 31), "stk_bn_stats_act: numel must be below 2^31");
  const uintptr_t align = uintptr_t(x) | uintptr_t(residual) | uintptr_t(weight) | uintptr_t(bias) | uintptr_t(out);
  STK_REQUIRE(c, align % 16 == 0, "stk_bn_stats_act: x, residual, weight, bias and out must be 16-byte aligned");
  DeviceGuard g(c->device);
  const uint32_t rows = uint32_t(numel / channels), groups = uint32_t(channels / 8);
  const BnBwdConfig cfg = bn_bwd_config(rows, uint32_t(channels));
  const bool bf16_run = running_dtype == STK_BF16;
  auto kern = two ? (bf16_run ? k_bn_stats_act<STK_ACT_RELU, true, __nv_bfloat16, true> : k_bn_stats_act<STK_ACT_RELU, true, float, true>)
              : bf16_run ? STK_BN_KERNEL(BnStatsKernel<__nv_bfloat16>::k, act, residual != nullptr)
                         : STK_BN_KERNEL(BnStatsKernel<float>::k, act, residual != nullptr);
  // as many blocks as the busiest phase uses, at most every resident one (the grid barriers need them all resident)
  const uint32_t gb = kBwdThreads / (kChains * cfg.block_y), cb = kBwdThreads / cfg.block_y;
  const size_t items = std::max(size_t((groups + gb - 1) / gb) * cfg.grid_y, size_t((channels + cb - 1) / cb));
  const uint32_t nvec = uint32_t(numel / 8);
  const size_t resident = size_t(blocks_per_sm(c, kern, kBwdThreads)) * c->sm_count;
  size_t blocks = std::min(resident, std::max(items, (size_t(nvec) + kBwdThreads - 1) / kBwdThreads));
  STK_REQUIRE(c, blocks * kBwdThreads >= groups, "stk_bn_stats_act: too many channels for one resident grid");
  BnStatsArgs a;
  a.x = static_cast<const uint4*>(x);
  a.r = static_cast<const uint4*>(residual);
  a.weight = static_cast<const __nv_bfloat16*>(weight);
  a.bias = static_cast<const __nv_bfloat16*>(bias);
  a.running_mean = running_mean;
  a.running_var = running_var;
  a.out = static_cast<uint4*>(out);
  a.save_mean = save_mean;
  a.save_invstd = save_invstd;
  a.ws = workspace;
  a.bar = c->grid_bar_dev;
  a.eps = float(eps);
  a.momentum = float(momentum);
  a.one_minus_momentum = 1.f - a.momentum;
  a.bessel = float(double(rows) / double(rows - 1));
  a.rows = rows;
  a.groups = groups;
  a.block_y = cfg.block_y;
  a.grid_y = cfg.grid_y;
  a.loops = cfg.loops;
  a.nvec = nvec;
  a.active = uint32_t(blocks * kBwdThreads / groups * groups);
  a.weight2 = static_cast<const __nv_bfloat16*>(weight2);
  a.bias2 = static_cast<const __nv_bfloat16*>(bias2);
  a.running_mean2 = running_mean2;
  a.running_var2 = running_var2;
  a.save_mean2 = save_mean2;
  a.save_invstd2 = save_invstd2;
  a.eps2 = float(eps2);
  a.momentum2 = float(momentum2);
  a.one_minus_momentum2 = 1.f - a.momentum2;
  cudaLaunchConfig_t lc{};
  lc.gridDim = dim3(unsigned(blocks));
  lc.blockDim = dim3(kBwdThreads);
  lc.stream = reinterpret_cast<cudaStream_t>(stream);
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = 1;
  lc.attrs = attr;
  lc.numAttrs = 1;
  STK_CUDA(c, cudaLaunchKernelEx(&lc, kern, a));
  return STK_OK;
}

int stk_bn_act(stk_ctx* c, const void* x, const void* residual, const float* mean, const float* var, const void* weight,
               const void* bias, double eps, void* out, float* save_invstd, size_t numel, size_t channels, void* stream) {
  return stk_bn_act_ex(c, STK_ACT_RELU, x, residual, mean, var, weight, bias, eps, out, save_invstd, numel, channels,
                       stream);
}

int stk_bn_act_backward_ex(stk_ctx* c, int act, const void* grad, const void* x, const void* out, const float* mean,
                           const float* invstd, const void* weight, const void* bias, void* grad_x, void* grad_weight,
                           void* grad_bias, void* grad_residual, void* grad_pre, float* workspace, size_t numel,
                           size_t channels, void* stream, const void* grad2, const void* x2, const float* mean2,
                           const float* invstd2, const void* weight2, void* grad_x2, void* grad_weight2,
                           void* grad_bias2) {
  STK_REQUIRE(c, c && grad && x && mean && invstd && weight && grad_weight && grad_bias && workspace,
              "stk_bn_act_backward: NULL argument");
  STK_REQUIRE(c, act_valid(act, out != nullptr),
              "stk_bn_act_backward: act must be an STK_ACT_* kind, and only STK_ACT_RELU takes a residual");
  STK_REQUIRE(c, out ? grad_residual != nullptr : bias != nullptr,
              "stk_bn_act_backward: a residual site needs grad_residual, a site without one needs bias");
  STK_REQUIRE(c, grad2 == nullptr || out != nullptr, "stk_bn_act_backward: only a residual site takes grad2");
  STK_REQUIRE(c, x2 == nullptr || (out && mean2 && invstd2 && weight2 && grad_weight2 && grad_bias2 &&
                                   (grad_x == nullptr) == (grad_x2 == nullptr)),
              "stk_bn_act_backward: x2 needs a residual site, mean2, invstd2, weight2, grad_weight2, grad_bias2, and "
              "grad_x2 exactly when grad_x");
  const uintptr_t align2 = uintptr_t(x2) | uintptr_t(mean2) | uintptr_t(invstd2) | uintptr_t(weight2) |
                           uintptr_t(grad_x2) | uintptr_t(grad_weight2) | uintptr_t(grad_bias2);
  STK_REQUIRE(c, align2 % 16 == 0, "stk_bn_act_backward: every tensor must be 16-byte aligned");
  STK_REQUIRE(c, grad_pre == nullptr || act != STK_ACT_RELU, "stk_bn_act_backward: grad_pre is not written for STK_ACT_RELU");
  STK_REQUIRE(c, channels > 0 && channels % 8 == 0 && numel % channels == 0 && numel >= channels,
              "stk_bn_act_backward: channels must be a positive multiple of 8 dividing numel");
  STK_REQUIRE(c, numel < (size_t(1) << 31), "stk_bn_act_backward: numel must be below 2^31");
  const uintptr_t align = uintptr_t(grad) | uintptr_t(x) | uintptr_t(out) | uintptr_t(mean) | uintptr_t(invstd) |
                          uintptr_t(weight) | uintptr_t(bias) | uintptr_t(grad_x) | uintptr_t(grad_weight) |
                          uintptr_t(grad_bias) | uintptr_t(grad_residual) | uintptr_t(grad_pre) | uintptr_t(workspace) |
                          uintptr_t(grad2);
  STK_REQUIRE(c, align % 16 == 0, "stk_bn_act_backward: every tensor must be 16-byte aligned");
  DeviceGuard g(c->device);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const uint32_t rows = uint32_t(numel / channels), groups = uint32_t(channels / 8);
  const BnBwdConfig cfg = bn_bwd_config(rows, uint32_t(channels));
  const bool res = out != nullptr;
  const uint32_t gb = kBwdThreads / (kChains * cfg.block_y);   // block_y <= 512 / 8 since channels >= 8
  const dim3 grid((groups + gb - 1) / gb, cfg.grid_y);
  const bool two = x2 != nullptr;
  BnBwdSecond s2{static_cast<const uint4*>(x2), mean2, invstd2, static_cast<const __nv_bfloat16*>(weight2),
                 workspace + 2 * channels * (1 + size_t(cfg.grid_y)), static_cast<__nv_bfloat16*>(grad_weight2),
                 static_cast<__nv_bfloat16*>(grad_bias2), static_cast<uint4*>(grad_x2)};
  auto reduce = two ? (grad2 ? k_bn_bwd_reduce<STK_ACT_RELU, true, true, true> : k_bn_bwd_reduce<STK_ACT_RELU, true, false, true>)
                : grad2 ? k_bn_bwd_reduce<STK_ACT_RELU, true, true>
                        : STK_BN_KERNEL(k_bn_bwd_reduce, act, res);
  auto bf = [](const void* p) { return static_cast<const __nv_bfloat16*>(p); };
  reduce<<<grid, kBwdThreads, 0, s>>>(static_cast<const uint4*>(grad), static_cast<const uint4*>(grad2),
                                      static_cast<const uint4*>(x),
                                      static_cast<const uint4*>(out), mean, invstd, bf(weight), bf(bias),
                                      static_cast<uint4*>(res ? grad_residual : grad_pre), workspace,
                                      static_cast<__nv_bfloat16*>(grad_weight), static_cast<__nv_bfloat16*>(grad_bias),
                                      rows, groups, cfg.block_y, cfg.loops, s2);
  STK_CUDA(c, cudaGetLastError());
  if (cfg.grid_y > 1) {
    const uint32_t cb = kBwdThreads / cfg.block_y;
    (two ? k_bn_bwd_finish<true> : k_bn_bwd_finish<false>)<<<unsigned((channels + cb - 1) / cb), kBwdThreads, 0, s>>>(
        workspace, invstd, static_cast<__nv_bfloat16*>(grad_weight), static_cast<__nv_bfloat16*>(grad_bias),
        uint32_t(channels), cfg.block_y, cfg.grid_y, s2);
    STK_CUDA(c, cudaGetLastError());
  }
  if (grad_x) {
    const uint32_t nvec = uint32_t(numel / 8);
    auto elemt = two ? k_bn_bwd_elemt<STK_ACT_RELU, true, true> : STK_BN_KERNEL(k_bn_bwd_elemt, act, res);
    const size_t resident = size_t(blocks_per_sm(c, elemt, kBnThreads)) * c->sm_count;
    size_t blocks = std::min(resident, (size_t(nvec) + kBnThreads - 1) / kBnThreads);
    blocks = std::max(blocks, (size_t(groups) + kBnThreads - 1) / kBnThreads);
    const uint32_t active = uint32_t(blocks * kBnThreads / groups * groups);
    elemt<<<unsigned(blocks), kBnThreads, 0, s>>>(static_cast<const uint4*>(res ? grad_residual : grad),
                                                  static_cast<const uint4*>(x), mean, invstd, bf(weight), bf(bias),
                                                  workspace, static_cast<uint4*>(grad_x), float(1.0 / double(rows)),
                                                  nvec, groups, active, s2);
    STK_CUDA(c, cudaGetLastError());
  }
  return STK_OK;
}

int stk_bn_act_backward(stk_ctx* c, const void* grad, const void* x, const void* out, const float* mean, const float* invstd,
                        const void* weight, const void* bias, void* grad_x, void* grad_weight, void* grad_bias,
                        void* grad_residual, float* workspace, size_t numel, size_t channels, void* stream) {
  return stk_bn_act_backward_ex(c, STK_ACT_RELU, grad, x, out, mean, invstd, weight, bias, grad_x, grad_weight, grad_bias,
                                grad_residual, nullptr, workspace, numel, channels, stream, nullptr, nullptr, nullptr,
                                nullptr, nullptr, nullptr, nullptr, nullptr);
}

}  // extern "C"
