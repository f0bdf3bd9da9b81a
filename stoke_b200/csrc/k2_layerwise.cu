// k2_layerwise.cu -- fused LAMB, LARS and StableAdamW steps (stoke_b200.optim.LAMB / LARS / StableAdamW): an
// element-wise update scaled by a per-parameter factor (a trust ratio, or StableAdamW's 1 / max(RMS, 1)), which needs
// whole-parameter sums before any element can be updated.  Three stream-ordered launches, no host involvement:
//
//   1 k_lw_tiles  tile pass (one block per kLwTile elements of one parameter), 16-byte vectors:
//                 LAMB: reads g, w, m, v; writes m, v; per-tile sums of w^2 and r^2; zeroes the raw bucket
//                 LARS: reads g, w; per-tile sums of w^2 and g^2
//                 StableAdamW: reads g, m, v; writes m, v; per-tile sum of g^2 / max(v, eps^2); zeroes the raw bucket
//   2 k_lw_fold   one warp per parameter: folds its tile partials in index order into the trust ratio (StableAdamW:
//                 lr_t); advances the step count; writes the per-parameter scalars of pass 3
//   3 k_lw_apply  tile pass: the update, the fp32 master and the low-precision copy
//                 LAMB: reads w, m, v and recomputes r with the same fp32 operations as pass 1 (bit-identical r)
//                 LARS: reads g, w, buf; writes buf; zeroes the raw bucket
//                 StableAdamW: reads w, m, v
//
// HBM bytes per element, world-1 bf16 raw route: LAMB 24 + 18 = 42, LARS 6 + 22 = 28 (momentum != 0), StableAdamW
// 20 + 18 = 38.
// Every sum adds in an order fixed by the shapes and these launch shapes only (a thread's vectors in index order, a
// fixed-tree block reduction, tile partials folded lane-strided then by a fixed shuffle tree), and nothing uses a
// floating-point atomic: two identical runs are bit-identical.  A skipped parameter (bit 7 of its group byte) or a step
// with found_inf leaves master, state and step count as they are; the raw bucket is zeroed all the same.
#include "k1_common.cuh"

namespace stk {

constexpr int kLwTile = STK_LW_TILE;   // elements per block of the tile passes
constexpr int kLwThreads = 256;

struct LwGroup {      // per group, converted once on the host (fp32 as the update uses them)
  double beta1, beta2;                  // LAMB's bias corrections are formed in double from these
  float lr, one_m_b1, b2, one_m_b2, eps, wd, mom, one_m_damp, tc;
  int bias_correction, nesterov, adapt;  // adapt: weight_decay != 0 or always_adapt
};
struct LwScal {       // per parameter, written by pass 2 for pass 3
  float trust, bc1, bc2;   // StableAdamW: trust = lr_t, bc1 = 1 - lr_t wd
  int flags;          // bit 0: stepped this step; bit 1: its first step (t == 1)
};

struct LwParams {
  const stk_layerwise_param_t* prm;
  int n_params;
  const uint8_t* pgroup;
  int32_t* steps;
  float* master;
  float* m;
  float* v;
  float2* part;       // per tile: {sum w^2, sum r^2 (LAMB) | sum g^2 (LARS)}
  LwScal* scal;
  const void* grad;
  const float* acc;
  void* lp;
  const stk_scaler_state_t* scaler;
  float grad_mul, clip_max_norm, clip_value;
  int raw, lp_dtype, clip_kind, kind;
  LwGroup g[STK_MAX_GROUPS];
  float eps_sq[STK_MAX_GROUPS];   // StableAdamW: fp32 of the python double eps * eps (after g: LAMB's and LARS's layout
                                  // of the fields above is theirs)
};

// largest j with tile0(prm[j]) <= tile: the parameter owning the tile (an empty parameter shares its tile0 with the next
// one, which then wins)
__device__ __forceinline__ int lw_find(const LwParams& p, int tile) {
  int lo = 0, hi = p.n_params - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (p.prm[mid].tile0 <= tile) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// LAMB's bias corrections of step t: python doubles 1 - beta^t, as fp32 operands of the tensor divisions
__device__ __forceinline__ float2 lw_bias(const LwGroup& h, int32_t t) {
  if (!h.bias_correction) return make_float2(1.f, 1.f);
  return make_float2((float)(1.0 - pow(h.beta1, (double)t)), (float)(1.0 - pow(h.beta2, (double)t)));
}

// LAMB's r = (m / bc1) / (sqrt(v / bc2) + eps) + wd w, with explicit rounding so that passes 1 and 3 form the same bits
__device__ __forceinline__ float lamb_r(float m, float v, float w, float bc1, float bc2, const LwGroup& h) {
  const float den = __fadd_rn(__fsqrt_rn(__fdiv_rn(v, bc2)), h.eps);
  return __fadd_rn(__fdiv_rn(__fdiv_rn(m, bc1), den), __fmul_rn(h.wd, w));
}

// StableAdamW's debiased betas of step t in python doubles, b = beta (1 - beta^(t-1)) / (1 - beta^t), as the fp32 scalar
// operands torch makes of them: {1 - b1 (lerp_'s weight), b2 (mul_), 1 - b2 (addcmul_'s value)}
__device__ __forceinline__ float3 sa_betas(const LwGroup& h, int32_t t) {
  const double b1 = h.beta1 * (1.0 - pow(h.beta1, (double)(t - 1))) / (1.0 - pow(h.beta1, (double)t));
  const double b2 = h.beta2 * (1.0 - pow(h.beta2, (double)(t - 1))) / (1.0 - pow(h.beta2, (double)t));
  return make_float3((float)(1.0 - b1), (float)b2, (float)(1.0 - b2));
}

// torch.clamp(x, min=lo): a NaN x stays NaN (fmaxf would give lo)
__device__ __forceinline__ float clamp_min_nan(float x, float lo) { return x < lo ? lo : x; }

struct LwGrad {        // what turns a stored gradient element into the optimizer's g (form_grad, shared with K2)
  float inv_scale, coef;
};
__device__ __forceinline__ LwGrad lw_grad_scalars(const LwParams& p) {
  return LwGrad{p.raw ? (float)(1.0 / (double)p.scaler->scale) : 1.f, clip_coef(p.clip_kind, p.clip_max_norm, p.scaler)};
}
// the 8 gradients of vector vi: raw bucket [+ accumulator] or fp32 main gradients, then form_grad
template <int GDT>
__device__ __forceinline__ void lw_load_grad(const LwParams& p, const LwGrad& s, size_t vi, float (&g)[8]) {
  InVec<GDT>::load(p.grad, vi, g);
  if (p.acc != nullptr) {
    float a[8];
    InVec<STK_F32>::load(p.acc, vi, a);
#pragma unroll
    for (int e = 0; e < 8; ++e) g[e] += a[e];
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) g[e] = form_grad(g[e], p.raw != 0, p.grad_mul, s.inv_scale, p.clip_kind, s.coef, p.clip_value);
}

// ---- 1: tile pass -----------------------------------------------------------------------------------------------------
template <int KIND, int GDT>
__global__ void __launch_bounds__(kLwThreads) k_lw_tiles(const LwParams p) {
  __shared__ float s_red[2][32];
  __shared__ float2 s_bc;
  __shared__ float3 s_sb;   // StableAdamW: sa_betas
  const int tile = blockIdx.x;
  const int j = lw_find(p, tile);
  const stk_layerwise_param_t d = p.prm[j];
  const unsigned gb = p.pgroup[j];
  const LwGroup& h = p.g[gb & 0x7f];
  const bool live = p.scaler->found_inf == 0 && !(gb & 0x80u);
  const int q0 = (tile - d.tile0) * kLwTile;
  const int nq = min(kLwTile, d.numel - q0);
  const int nvec = (nq + 7) >> 3;
  const size_t v0 = (d.offset + (size_t)q0) >> 3;
  if constexpr (KIND == STK_LW_LARS) {
    if (!live || !h.adapt) return;   // nothing to reduce (pass 3 reads and zeroes the bucket)
  } else {
    if (!live) {                     // the bucket is consumed here: zero it also on a skipped step
      if (p.raw)
        for (int k = threadIdx.x; k < nvec; k += kLwThreads) InVec<GDT>::zero(const_cast<void*>(p.grad), v0 + k);
      return;
    }
    if (threadIdx.x == 0) {
      if constexpr (KIND == STK_LW_LAMB) s_bc = lw_bias(h, p.steps[j] + 1);
      else s_sb = sa_betas(h, p.steps[j] + 1);
    }
    __syncthreads();
  }
  const LwGrad f = lw_grad_scalars(p);
  float sw = 0.f, sx = 0.f;
  for (int k = threadIdx.x; k < nvec; k += kLwThreads) {
    const size_t vi = v0 + k;
    const int valid = min(8, nq - 8 * k);   // the parameter's last vector may end in padding: left untouched
    float g[8], w[8];
    lw_load_grad<GDT>(p, f, vi, g);
    if constexpr (KIND == STK_LW_STABLE_ADAMW) {
      float m[8], v[8];
      InVec<STK_F32>::load(p.m, vi, m);
      InVec<STK_F32>::load(p.v, vi, v);
      const float3 sb = s_sb;
      const float e2 = p.eps_sq[gb & 0x7f];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        if (e >= valid) continue;
        const float gg = g[e], g2 = __fmul_rn(gg, gg);
        m[e] = lerp_torch(m[e], gg, sb.x);                   // exp_avg.lerp_(g, 1 - b1)
        // exp_avg_sq.mul_(b2).addcmul_(g, g, value=1 - b2): Tensor.addcmul_ rounds g * g first, then one FFMA (K2's
        // foreach form, fma((1 - b2) g, g, .), rounds (1 - b2) g instead)
        v[e] = fmaf(sb.z, g2, v[e] * sb.y);
        sw += __fdiv_rn(g2, clamp_min_nan(v[e], e2));        // (g * g).div_(v.clamp(min=eps * eps))
      }
      st_stream_f8(p.m + vi * 8, m);
      st_stream_f8(p.v + vi * 8, v);
      if (p.raw) InVec<GDT>::zero(const_cast<void*>(p.grad), vi);
      continue;
    }
    InVec<STK_F32>::load(p.master, vi, w);
    if constexpr (KIND == STK_LW_LAMB) {
      float m[8], v[8];
      InVec<STK_F32>::load(p.m, vi, m);
      InVec<STK_F32>::load(p.v, vi, v);
      const float2 bc = s_bc;
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        if (e >= valid) continue;
        const float gg = g[e];
        m[e] = fmaf(h.one_m_b1, gg - m[e], m[e]);            // exp_avg.lerp_(g, 1 - beta1)
        v[e] = fmaf(h.one_m_b2 * gg, gg, v[e] * h.b2);       // exp_avg_sq.mul_(beta2).addcmul_(g, g, value=1 - beta2)
        if (h.adapt) {
          const float r = lamb_r(m[e], v[e], w[e], bc.x, bc.y, h);
          sw = fmaf(w[e], w[e], sw);
          sx = fmaf(r, r, sx);
        }
      }
      st_stream_f8(p.m + vi * 8, m);
      st_stream_f8(p.v + vi * 8, v);
      if (p.raw) InVec<GDT>::zero(const_cast<void*>(p.grad), vi);
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        if (e >= valid) continue;
        sw = fmaf(w[e], w[e], sw);
        sx = fmaf(g[e], g[e], sx);
      }
    }
  }
  if (KIND == STK_LW_LAMB && !h.adapt) return;   // uniform per block
  if constexpr (KIND == STK_LW_STABLE_ADAMW) {
    sw = block_reduce<false>(sw, s_red[0]);
    if (threadIdx.x == 0) p.part[tile] = make_float2(sw, 0.f);
    return;
  }
  sw = block_reduce<false>(sw, s_red[0]);
  sx = block_reduce<false>(sx, s_red[1]);
  if (threadIdx.x == 0) p.part[tile] = make_float2(sw, sx);
}

// ---- 2: per-parameter fold: trust ratio, step count ---------------------------------------------------------------------
__global__ void __launch_bounds__(kLwThreads) k_lw_fold(const LwParams p) {
  const int j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (j >= p.n_params) return;   // whole warp
  const stk_layerwise_param_t& d = p.prm[j];
  const unsigned gb = p.pgroup[j];
  const LwGroup& h = p.g[gb & 0x7f];
  const bool live = p.scaler->found_inf == 0 && !(gb & 0x80u);
  const int ntile = (d.numel + kLwTile - 1) / kLwTile;
  float sw = 0.f, sx = 0.f;
  if (live && (h.adapt || p.kind == STK_LW_STABLE_ADAMW))
    for (int k = lane; k < ntile; k += 32) {
      const float2 t = p.part[d.tile0 + k];
      sw += t.x;
      sx += t.y;
    }
  sw = warp_reduce<false>(sw);
  sx = warp_reduce<false>(sx);
  if (lane != 0) return;
  LwScal o{1.f, 1.f, 1.f, 0};
  if (live) {
    const int32_t t = p.steps[j] + 1;
    if (p.kind == STK_LW_STABLE_ADAMW) {
      // rms = sqrt(mean(g^2 / max(v, eps^2))); lr_t = rms.clamp(min=1).reciprocal() * lr: a NaN rms gives a NaN lr_t
      const float rms = __fsqrt_rn(__fdiv_rn(sw, (float)d.numel));
      o.trust = __fmul_rn(__frcp_rn(clamp_min_nan(rms, 1.f)), h.lr);
      o.bc1 = __fsub_rn(1.f, __fmul_rn(o.trust, h.wd));   // 1 - lr_t * weight_decay
    } else if (h.adapt) {
      // torch.where semantics: a comparison with a NaN norm is false, so the trust ratio is 1 then
      const float wn = sqrtf(sw), xn = sqrtf(sx);
      if (p.kind == STK_LW_LAMB) {
        if (wn > 0.f && xn > 0.f) o.trust = __fdiv_rn(wn, xn);                         // ||w|| / ||r||
      } else if (wn > 0.f && xn > 0.f) {                                              // tc ||w|| / (||g|| + wd ||w|| + eps)
        o.trust = __fdiv_rn(__fmul_rn(h.tc, wn), __fadd_rn(__fadd_rn(xn, __fmul_rn(h.wd, wn)), h.eps));
      }
    }
    if (p.kind == STK_LW_LAMB) {
      const float2 bc = lw_bias(h, t);
      o.bc1 = bc.x;
      o.bc2 = bc.y;
    }
    o.flags = 1 | (t == 1 ? 2 : 0);
    p.steps[j] = t;
  }
  p.scal[j] = o;
}

// ---- 3: the update, the low-precision copy --------------------------------------------------------------------------------
template <int KIND, int GDT>
__global__ void __launch_bounds__(kLwThreads) k_lw_apply(const LwParams p) {
  const int tile = blockIdx.x;
  const int j = lw_find(p, tile);
  const stk_layerwise_param_t d = p.prm[j];
  const LwGroup& h = p.g[p.pgroup[j] & 0x7f];
  const LwScal sc = p.scal[j];
  const int q0 = (tile - d.tile0) * kLwTile;
  const int nq = min(kLwTile, d.numel - q0);
  const int nvec = (nq + 7) >> 3;
  const size_t v0 = (d.offset + (size_t)q0) >> 3;
  const bool live = sc.flags & 1;
  if (KIND != STK_LW_LARS && !live) return;
  const LwGrad f = lw_grad_scalars(p);
  const bool first = sc.flags & 2;
  for (int k = threadIdx.x; k < nvec; k += kLwThreads) {
    const size_t vi = v0 + k;
    if (live) {
      const int valid = min(8, nq - 8 * k);
      float w[8];
      InVec<STK_F32>::load(p.master, vi, w);
      if constexpr (KIND == STK_LW_LAMB) {
        float m[8], v[8];
        InVec<STK_F32>::load(p.m, vi, m);
        InVec<STK_F32>::load(p.v, vi, v);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          if (e >= valid) continue;
          const float r = lamb_r(m[e], v[e], w[e], sc.bc1, sc.bc2, h);
          w[e] = fmaf(-h.lr, __fmul_rn(sc.trust, r), w[e]);   // param.add_(trust * r, alpha=-lr)
        }
      } else if constexpr (KIND == STK_LW_STABLE_ADAMW) {
        float m[8], v[8];
        InVec<STK_F32>::load(p.m, vi, m);
        InVec<STK_F32>::load(p.v, vi, v);
        const bool decay = h.wd != 0.f;
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          if (e >= valid) continue;
          float ww = w[e];
          if (decay) ww = __fmul_rn(ww, sc.bc1);                                  // w.mul_(1 - lr_t * wd)
          const float u = __fdiv_rn(m[e], __fadd_rn(__fsqrt_rn(v[e]), h.eps));   // m / (v.sqrt() + eps)
          w[e] = __fsub_rn(ww, __fmul_rn(sc.trust, u));                           // w.sub_(lr_t * u)
        }
      } else {
        float g[8], b[8];
        lw_load_grad<GDT>(p, f, vi, g);
        const bool mom = h.mom != 0.f;
        if (mom && !first) InVec<STK_F32>::load(p.m, vi, b);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          if (e >= valid) continue;
          float gg = g[e];
          if (h.adapt) gg = __fmul_rn(fmaf(h.wd, w[e], gg), sc.trust);      // (g + wd w) * trust
          if (mom) {
            b[e] = first ? gg : fmaf(b[e], h.mom, h.one_m_damp * gg);    // first step: buf = g (torch's SGD seeding)
            gg = h.nesterov ? fmaf(b[e], h.mom, gg) : b[e];
          }
          w[e] = fmaf(-h.lr, gg, w[e]);
        }
        if (mom) {
          if (first)   // the padding of a first buffer is zero, like the rest of the fresh state
#pragma unroll
            for (int e = 0; e < 8; ++e)
              if (e >= valid) b[e] = 0.f;
          st_stream_f8(p.m + vi * 8, b);
        }
      }
      st_stream_f8(p.master + vi * 8, w);
      if (p.lp != nullptr) {
        if (p.lp_dtype == STK_BF16) store_out<STK_BF16>(p.lp, vi, w);
        else store_out<STK_F32>(p.lp, vi, w);
      }
    }
    if (KIND == STK_LW_LARS && p.raw) InVec<GDT>::zero(const_cast<void*>(p.grad), vi);
  }
}

template <int KIND, int GDT>
void lw_launch(const LwParams& p, int n_tiles, unsigned warps_grid, cudaStream_t s) {
  k_lw_tiles<KIND, GDT><<<n_tiles, kLwThreads, 0, s>>>(p);
  k_lw_fold<<<warps_grid, kLwThreads, 0, s>>>(p);
  k_lw_apply<KIND, GDT><<<n_tiles, kLwThreads, 0, s>>>(p);
}

}  // namespace stk

using namespace stk;

extern "C" {

int stk_layerwise_step(stk_ctx* c, const stk_layerwise_args_t* a, void* stream) {
  STK_REQUIRE(c, c && a && a->hyper && a->params && a->param_group && a->steps && a->master && a->workspace && a->grad,
              "stk_layerwise_step: NULL argument");
  STK_REQUIRE(c, a->kind == STK_LW_LAMB || a->kind == STK_LW_LARS || a->kind == STK_LW_STABLE_ADAMW,
              "stk_layerwise_step: kind");
  STK_REQUIRE(c, a->n_groups >= 1 && a->n_groups <= STK_MAX_GROUPS, "stk_layerwise_step: n_groups must be in [1, 8]");
  STK_REQUIRE(c, a->n_params >= 1 && a->n_tiles >= 1, "stk_layerwise_step: no parameters");
  STK_REQUIRE(c, (reinterpret_cast<uintptr_t>(a->workspace) & 15) == 0, "stk_layerwise_step: workspace must be 16-byte aligned");
  STK_REQUIRE(c, a->grad_raw ? (a->grad_dtype == STK_BF16 || a->grad_dtype == STK_F32) : a->grad_dtype == STK_F32,
              "stk_layerwise_step: gradients must be a bf16 / fp32 raw bucket or fp32 main gradients");
  STK_REQUIRE(c, a->lp == nullptr || a->lp_dtype == STK_BF16 || a->lp_dtype == STK_F32, "stk_layerwise_step: lp dtype");
  STK_REQUIRE(c, a->clip_kind >= STK_CLIP_NONE && a->clip_kind <= STK_CLIP_VALUE, "stk_layerwise_step: clip kind");
  bool any_mom = false;
  for (int gi = 0; gi < a->n_groups; ++gi) any_mom |= a->hyper[gi].momentum != 0.0;
  STK_REQUIRE(c, a->kind == STK_LW_LARS ? (!any_mom || a->exp_avg) : (a->exp_avg && a->exp_avg_sq),
              "stk_layerwise_step: LAMB and StableAdamW need exp_avg and exp_avg_sq, LARS with momentum needs exp_avg");
  std::lock_guard<std::mutex> lk(c->mu);
  DeviceGuard g(c->device);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);

  LwParams p{};
  p.prm = a->params;
  p.n_params = a->n_params;
  p.pgroup = a->param_group;
  p.steps = a->steps;
  p.master = a->master;
  p.m = a->exp_avg;
  p.v = a->exp_avg_sq;
  p.scal = reinterpret_cast<LwScal*>(a->workspace);
  p.part = reinterpret_cast<float2*>(static_cast<char*>(a->workspace) + size_t(a->n_params) * sizeof(LwScal));
  p.grad = a->grad;
  p.acc = a->grad_raw ? a->acc : nullptr;
  p.lp = a->lp;
  p.scaler = c->scaler_dev;
  p.grad_mul = (float)a->grad_mul;
  p.clip_max_norm = (float)a->clip_max_norm;
  p.clip_value = (float)a->clip_value;
  p.raw = a->grad_raw ? 1 : 0;
  p.lp_dtype = a->lp_dtype;
  p.clip_kind = a->clip_kind;
  p.kind = a->kind;
  for (int gi = 0; gi < a->n_groups; ++gi) {
    const stk_layerwise_hyper_t& h = a->hyper[gi];
    LwGroup& o = p.g[gi];
    o.beta1 = h.beta1;
    o.beta2 = h.beta2;
    o.lr = (float)h.lr;
    o.one_m_b1 = (float)(1.0 - h.beta1);
    o.b2 = (float)h.beta2;
    o.one_m_b2 = (float)(1.0 - h.beta2);
    o.eps = (float)h.eps;
    o.wd = (float)h.weight_decay;
    o.mom = (float)h.momentum;
    o.one_m_damp = (float)(1.0 - h.dampening);
    o.tc = (float)h.trust_coefficient;
    o.bias_correction = h.bias_correction;
    o.nesterov = h.nesterov;
    o.adapt = h.weight_decay != 0.0 || h.always_adapt;
    p.eps_sq[gi] = (float)(h.eps * h.eps);
  }
  const unsigned warps_grid = (unsigned)((32ll * a->n_params + kLwThreads - 1) / kLwThreads);
  const bool bf16 = a->grad_raw && a->grad_dtype == STK_BF16;
  ProfScope prof(c, 1, s);
  if (a->kind == STK_LW_LAMB) {
    if (bf16) lw_launch<STK_LW_LAMB, STK_BF16>(p, a->n_tiles, warps_grid, s);
    else lw_launch<STK_LW_LAMB, STK_F32>(p, a->n_tiles, warps_grid, s);
  } else if (a->kind == STK_LW_LARS) {
    if (bf16) lw_launch<STK_LW_LARS, STK_BF16>(p, a->n_tiles, warps_grid, s);
    else lw_launch<STK_LW_LARS, STK_F32>(p, a->n_tiles, warps_grid, s);
  } else {
    if (bf16) lw_launch<STK_LW_STABLE_ADAMW, STK_BF16>(p, a->n_tiles, warps_grid, s);
    else lw_launch<STK_LW_STABLE_ADAMW, STK_F32>(p, a->n_tiles, warps_grid, s);
  }
  STK_CUDA(c, cudaGetLastError());
  return STK_OK;
}

}  // extern "C"
