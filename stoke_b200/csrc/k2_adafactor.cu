// k2_adafactor.cu -- fused torch.optim.Adafactor step (torch/optim/_adafactor.py, _single_tensor_adafactor).
//
// Adafactor cannot be another kind of k_optim_step: its update needs per-parameter reductions (row and column means of g^2,
// the parameter's RMS, the RMS of the update, which feeds a clip).  Eight stream-ordered launches, no host involvement:
//
//   1 k_af_sumsq_w      tile pass (one block per TILE elements of one parameter): per-tile sum w^2
//   2 k_af_prologue     one warp per parameter: folds the tiles of ||w||^2; b2hat, rho, alpha in double from torch's
//                       python-scalar formulas; the step count advance
//   3 k_af_lines        one thread per (row or column, CHUNK elements): partial sums of g^2
//   4 k_af_lines_finish one thread per row / column: folds its chunks in order; lerp_ of row_var / col_var
//   5 k_af_rowmean      one thread (R <= 32) or one warp (R > 32) per batch index b: clamp_min(mean_r row_var, eps1)
//   6 k_af_unorm        tile pass: u = g rsqrt(clamp_min(v, eps1^2)) and per-tile sum u^2 (vectors: variance.lerp_ here)
//   7 k_af_coef         one warp per parameter: -alpha / max(1, ||u|| / (sqrt(numel) d))
//   8 k_af_apply        tile pass: w = w (1 - lr wd) + coef u, the fp32 master and the low-precision copy; zeroes the raw
//                       bucket (also on a skipped step)
//
// Every sum adds in an order fixed by the shapes and these launch shapes only (fixed-tree block / warp reductions, chunk
// and tile partials folded in index order): two identical runs are bit-identical.  Every pass forms the same fp32 gradient
// (raw bucket [+ accumulator] * grad_mul * 1/scale, then the clip exactly as k_optim_step forms it).  A parameter is mapped
// from its storage position to its logical (b, r, c) through its sizes and strides, so channels-last weights keep torch's
// factorisation over their last two logical dims.
#include <cfloat>

#include "k1_common.cuh"

namespace stk {

constexpr int kAfTile = 8192;     // elements per block of the tile passes
constexpr int kAfChunk = 32;      // elements per partial of a row / column sum
constexpr int kAfThreads = 256;

struct AfGroup {
  double lr, beta2_decay, eps1, eps2, d, weight_decay;
  int eps1_none, maximize;
};
struct AfScal {       // per-parameter scalars of this step (workspace)
  double alpha;
  float b2hat, decay, coef, eps1, eps1sq;
  int live;           // stepped this step (has a gradient, no found_inf)
  int wd, maximize;
};

struct AfParams {
  const stk_adafactor_param_t* prm;
  int n_params;
  const uint8_t* pgroup;
  int32_t* steps;
  float* master;
  float* state;
  float *part_w, *part_u, *line, *rmean;
  AfScal* scal;
  const void* grad;
  const float* acc;
  void* lp;
  const stk_scaler_state_t* scaler;
  float grad_mul, clip_max_norm, clip_value;
  int grad_dtype, raw, lp_dtype, clip_kind;
  int n_tiles;
  long long n_line, n_out, n_rm;
  int n_groups;
  AfGroup g[STK_MAX_GROUPS];
};

// largest j with start(prm[j]) <= x: the parameter owning item x (parameters without items of this kind share their start
// with the next one, which then wins)
template <typename F>
__device__ __forceinline__ int af_find(const AfParams& p, long long x, F start) {
  int lo = 0, hi = p.n_params - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (start(p.prm[mid]) <= x) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

struct AfGrad {       // what turns a stored gradient element into torch's g
  float mul, inv_scale, coef;
};
__device__ __forceinline__ AfGrad af_grad_scalars(const AfParams& p) {
  AfGrad s;
  s.mul = p.grad_mul;
  s.inv_scale = p.raw ? (float)(1.0 / (double)p.scaler->scale) : 1.f;
  s.coef = p.clip_kind == STK_CLIP_NORM ? clamp_max_nan(p.clip_max_norm / (p.scaler->grad_norm + 1e-6f), 1.0f) : 1.f;
  return s;
}
// the fp32 gradient of flat element i, after unscale / accumulate / clip (maximize is applied by the caller), formed
// exactly as k_optim_step forms it
__device__ __forceinline__ float af_g(const AfParams& p, const AfGrad& s, size_t i) {
  float g;
  if (p.raw) {
    if (p.grad_dtype == STK_BF16) g = __uint_as_float(uint32_t(reinterpret_cast<const unsigned short*>(p.grad)[i]) << 16);
    else g = reinterpret_cast<const float*>(p.grad)[i];
    if (p.acc != nullptr) g += p.acc[i];
    g *= s.mul;
    g *= s.inv_scale;
  } else {
    g = reinterpret_cast<const float*>(p.grad)[i];
  }
  if (p.clip_kind == STK_CLIP_NORM) g *= s.coef;
  else if (p.clip_kind == STK_CLIP_VALUE) g = clamp_nan(g, -p.clip_value, p.clip_value);
  return g;
}

__device__ __forceinline__ float clamp_min_nan(float x, float lo) { return x < lo ? lo : x; }  // torch.clamp: NaN stays

// torch's lerp (aten/src/ATen/native/Lerp.h) with a scalar weight
__device__ __forceinline__ float af_lerp(float self, float end, float w) {
  const float diff = end - self;
  return fabsf(w) < 0.5f ? fmaf(w, diff, self) : fmaf(-diff, 1.f - w, end);
}

// v of element q (storage position inside the parameter) of a factored parameter
__device__ __forceinline__ float af_v_factored(const AfParams& p, const stk_adafactor_param_t& d, uint32_t q) {
  const uint32_t B1 = d.size[1], R = d.size[2], C = d.size[3];
  uint32_t b, r, c;
  if (d.contiguous) {
    c = q % C;
    const uint32_t row = q / C;
    b = row / R;
    r = row - b * R;
  } else {
    const uint32_t i0 = d.size[0] > 1 ? (q / (uint32_t)d.stride[0]) % (uint32_t)d.size[0] : 0u;
    const uint32_t i1 = B1 > 1 ? (q / (uint32_t)d.stride[1]) % B1 : 0u;
    r = R > 1 ? (q / (uint32_t)d.stride[2]) % R : 0u;
    c = C > 1 ? (q / (uint32_t)d.stride[3]) % C : 0u;
    b = i0 * B1 + i1;
  }
  const float* st = p.state + d.state;
  const size_t nr = size_t(d.size[0]) * B1 * R;
  // var_estimate = row_var @ col_var, then .div_(row_var.mean(dim=-2).clamp_(min=eps1))
  return (st[size_t(b) * R + r] * st[nr + size_t(b) * C + c]) / p.rmean[d.b0 + b];
}

// ---- 1: per-tile sum of w^2 ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kAfThreads) k_af_sumsq_w(const AfParams p) {
  __shared__ float s_red[32];
  const int tile = blockIdx.x;
  const int j = af_find(p, tile, [](const stk_adafactor_param_t& d) { return (long long)d.tile0; });
  if (p.scaler->found_inf != 0 || (p.pgroup[j] & 0x80u)) return;  // uniform per block
  const stk_adafactor_param_t& d = p.prm[j];
  const int q0 = (tile - d.tile0) * kAfTile;
  const int q1 = min(q0 + kAfTile, d.numel);
  const float* w = p.master + d.offset;
  float s = 0.f;
  for (int q = q0 + threadIdx.x; q < q1; q += blockDim.x) s = fmaf(w[q], w[q], s);
  s = block_reduce<false>(s, s_red);
  if (threadIdx.x == 0) p.part_w[tile] = s;
}

// ---- 2: per-parameter scalars and the step count -------------------------------------------------------------------------
__global__ void k_af_prologue(const AfParams p) {
  const int j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (j >= p.n_params) return;  // whole warp
  const stk_adafactor_param_t& d = p.prm[j];
  const unsigned gb = p.pgroup[j];
  const bool live = p.scaler->found_inf == 0 && !(gb & 0x80u);
  const int ntile = (d.numel + kAfTile - 1) / kAfTile;
  float s = 0.f;
  if (live)
    for (int k = lane; k < ntile; k += 32) s += p.part_w[d.tile0 + k];
  s = warp_reduce<false>(s);
  if (lane != 0) return;
  const AfGroup& h = p.g[gb & 0x7f];
  AfScal o{};
  o.live = live ? 1 : 0;
  o.wd = h.weight_decay != 0.0;
  o.maximize = h.maximize;
  if (live) {
    const int32_t done = p.steps[j];
    const double t = (double)(done + 1);
    const double inv_sqrt_t = 1.0 / pow(t, 0.5);
    const double rho = inv_sqrt_t < h.lr ? inv_sqrt_t : h.lr;               // python min(lr, 1 / t ** 0.5)
    const double rms = (double)sqrtf(s) / sqrt((double)d.numel);           // param.norm(2).item() / numel ** 0.5
    o.alpha = (rms > h.eps2 ? rms : h.eps2) * rho;                          // python max(eps2, rms): NaN gives eps2
    o.b2hat = (float)pow(t, h.beta2_decay);
    o.decay = (float)(1.0 - h.lr * h.weight_decay);
    const double eps1 = h.eps1_none ? (double)FLT_EPSILON : h.eps1;         // torch.finfo(fp32 master).eps
    o.eps1 = (float)eps1;
    o.eps1sq = (float)(eps1 * eps1);
    p.steps[j] = done + 1;
  }
  p.scal[j] = o;
}

// ---- 3: chunk partials of the row / column sums of g^2 -------------------------------------------------------------------
// Items of a factored parameter: rows first (chunk-major: item = chunk * B*R + o), then columns (chunk * B*C + o).
__global__ void __launch_bounds__(kAfThreads) k_af_lines(const AfParams p) {
  const long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= p.n_line) return;
  const int j = af_find(p, w, [](const stk_adafactor_param_t& d) { return (long long)d.line0; });
  if (!p.scal[j].live) return;
  const stk_adafactor_param_t& d = p.prm[j];
  const AfGrad gs = af_grad_scalars(p);
  const long long B1 = d.size[1], R = d.size[2], C = d.size[3], B = d.size[0] * B1;
  const long long n_r = B * R, items_r = n_r * ((C + kAfChunk - 1) / kAfChunk);
  long long li = w - d.line0, base, b;
  int L, es, chunk;
  if (li < items_r) {
    chunk = (int)(li / n_r);
    const long long o = li % n_r;
    b = o / R;
    base = (o % R) * d.stride[2];
    L = (int)C;
    es = d.stride[3];
  } else {
    li -= items_r;
    const long long n_c = B * C;
    chunk = (int)(li / n_c);
    const long long o = li % n_c;
    b = o / C;
    base = (o % C) * d.stride[3];
    L = (int)R;
    es = d.stride[2];
  }
  base += (b / B1) * d.stride[0] + (b % B1) * d.stride[1];
  const int k0 = chunk * kAfChunk, k1 = min(k0 + kAfChunk, L);
  float s = 0.f;
  for (int k = k0; k < k1; ++k) {
    const float g = af_g(p, gs, d.offset + size_t(base + (long long)k * es));
    s = fmaf(g, g, s);
  }
  p.line[w] = s;
}

// ---- 4: row / column means and their lerp_ ------------------------------------------------------------------------------
__global__ void __launch_bounds__(kAfThreads) k_af_lines_finish(const AfParams p) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= p.n_out) return;
  const int j = af_find(p, o, [](const stk_adafactor_param_t& d) { return d.out0; });
  const AfScal sc = p.scal[j];
  if (!sc.live) return;
  const stk_adafactor_param_t& d = p.prm[j];
  const long long R = d.size[2], C = d.size[3], B = (long long)d.size[0] * d.size[1];
  const long long n_r = B * R, li = o - d.out0;
  long long idx, step_;
  int nch, L;
  if (li < n_r) {  // row (b, r): mean over c
    nch = (int)((C + kAfChunk - 1) / kAfChunk);
    idx = d.line0 + li;
    step_ = n_r;
    L = (int)C;
  } else {         // column (b, c): mean over r
    nch = (int)((R + kAfChunk - 1) / kAfChunk);
    idx = d.line0 + n_r * ((C + kAfChunk - 1) / kAfChunk) + (li - n_r);
    step_ = B * C;
    L = (int)R;
  }
  float s = 0.f;
  for (int k = 0; k < nch; ++k) s += p.line[idx + k * step_];
  float* st = p.state + d.state + li;   // row_var [B*R] then col_var [B*C]
  *st = af_lerp(*st, s / (float)L, sc.b2hat);
}

// ---- 5: clamp_min(mean_r row_var, eps1) per batch index ----------------------------------------------------------------
// Items: R <= 32 -> one per b (a thread sums its row_var[b, :] in order); R > 32 -> 32 per b (a warp, lane-strided, then a
// fixed shuffle tree), starting on a multiple of 32.
__global__ void __launch_bounds__(kAfThreads) k_af_rowmean(const AfParams p) {
  const long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= p.n_rm) return;
  const int j = af_find(p, w, [](const stk_adafactor_param_t& d) { return d.rm0; });
  const stk_adafactor_param_t& d = p.prm[j];
  const int R = d.size[2];
  const long long B = (long long)d.size[0] * d.size[1];
  const bool warp = R > 32;
  const long long li = w - d.rm0;
  if (!d.factored || li >= (warp ? 32 * B : B)) return;  // alignment gap (never inside a warp-mode warp)
  const AfScal sc = p.scal[j];
  if (!sc.live) return;  // uniform per parameter
  const float* rv = p.state + d.state;
  float s = 0.f;
  long long b;
  if (!warp) {
    b = li;
    for (int r = 0; r < R; ++r) s += rv[b * R + r];
  } else {
    b = li >> 5;
    for (int r = (int)(li & 31); r < R; r += 32) s += rv[b * R + r];
    s = warp_reduce<false>(s);
    if ((li & 31) != 0) return;
  }
  p.rmean[d.b0 + b] = clamp_min_nan(s / (float)R, sc.eps1);
}

// u of element q; vectors: kFirst forms variance.lerp_(g^2, b2hat) and writes it back, later passes read it
template <bool kFirst>
__device__ __forceinline__ float af_u(const AfParams& p, const stk_adafactor_param_t& d, const AfScal& sc, uint32_t q,
                                      float g) {
  float v;
  if (d.factored) {
    v = af_v_factored(p, d, q);
  } else {
    float* st = p.state + d.state + q;
    if (kFirst) {
      v = af_lerp(*st, g * g, sc.b2hat);
      *st = v;
    } else {
      v = *st;
    }
  }
  // update = var_estimate.clamp_(min=eps1 * eps1).rsqrt_(); update.mul_(grad)
  return (1.0f / sqrtf(clamp_min_nan(v, sc.eps1sq))) * g;
}

// ---- 6: per-tile sum of u^2 ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kAfThreads) k_af_unorm(const AfParams p) {
  __shared__ float s_red[32];
  const int tile = blockIdx.x;
  const int j = af_find(p, tile, [](const stk_adafactor_param_t& d) { return (long long)d.tile0; });
  const AfScal sc = p.scal[j];
  if (!sc.live) return;
  const stk_adafactor_param_t d = p.prm[j];
  const AfGrad gs = af_grad_scalars(p);
  const int q0 = (tile - d.tile0) * kAfTile;
  const int q1 = min(q0 + kAfTile, d.numel);
  float s = 0.f;
  for (int q = q0 + threadIdx.x; q < q1; q += blockDim.x) {
    float g = af_g(p, gs, d.offset + q);
    if (sc.maximize) g = -g;
    const float u = af_u<true>(p, d, sc, (uint32_t)q, g);
    s = fmaf(u, u, s);
  }
  s = block_reduce<false>(s, s_red);
  if (threadIdx.x == 0) p.part_u[tile] = s;
}

// ---- 7: the update coefficient ------------------------------------------------------------------------------------------------
__global__ void k_af_coef(const AfParams p) {
  const int j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (j >= p.n_params) return;
  if (!p.scal[j].live) return;  // whole warp
  const stk_adafactor_param_t& d = p.prm[j];
  const int ntile = (d.numel + kAfTile - 1) / kAfTile;
  float s = 0.f;
  for (int k = lane; k < ntile; k += 32) s += p.part_u[d.tile0 + k];
  s = warp_reduce<false>(s);
  if (lane != 0) return;
  const AfGroup& h = p.g[p.pgroup[j] & 0x7f];
  const double x = (double)sqrtf(s) / (sqrt((double)d.numel) * h.d);   // update.norm(2).item() / (numel ** 0.5 * d)
  const double denom = x > 1.0 ? x : 1.0;                                // python max(1.0, x): NaN gives 1
  p.scal[j].coef = (float)(-p.scal[j].alpha / denom);
}

// ---- 8: the update, the low-precision copy, the bucket zeroing ---------------------------------------------------------------
__global__ void __launch_bounds__(kAfThreads) k_af_apply(const AfParams p) {
  const int tile = blockIdx.x;
  const int j = af_find(p, tile, [](const stk_adafactor_param_t& d) { return (long long)d.tile0; });
  const stk_adafactor_param_t d = p.prm[j];
  const int q0 = (tile - d.tile0) * kAfTile;
  const int q1 = min(q0 + kAfTile, d.numel);
  const AfScal sc = p.scal[j];
  if (sc.live) {
    const AfGrad gs = af_grad_scalars(p);
    for (int q = q0 + threadIdx.x; q < q1; q += blockDim.x) {
      const size_t i = d.offset + q;
      float g = af_g(p, gs, i);
      if (sc.maximize) g = -g;
      const float u = af_u<false>(p, d, sc, (uint32_t)q, g);
      float w = p.master[i];
      if (sc.wd) w *= sc.decay;       // param.mul_(1 - lr * weight_decay)
      w = fmaf(sc.coef, u, w);        // param.add_(update, alpha=-alpha / denom)
      p.master[i] = w;
      if (p.lp != nullptr) {
        if (p.lp_dtype == STK_BF16) reinterpret_cast<__nv_bfloat16*>(p.lp)[i] = __float2bfloat16_rn(w);
        else reinterpret_cast<float*>(p.lp)[i] = w;
      }
    }
  }
  if (p.raw) {  // the bucket is consumed (also on a skipped step): zero it for the next backward's accumulation
    for (int q = q0 + threadIdx.x; q < q1; q += blockDim.x) {
      const size_t i = d.offset + q;
      if (p.grad_dtype == STK_BF16) reinterpret_cast<unsigned short*>(const_cast<void*>(p.grad))[i] = 0;
      else reinterpret_cast<float*>(const_cast<void*>(p.grad))[i] = 0.f;
    }
  }
}

}  // namespace stk

using namespace stk;

namespace {
size_t align16(size_t x) { return (x + 15) & ~size_t(15); }
}

extern "C" {

int stk_adafactor_plan(stk_adafactor_param_t* prm, int n, stk_adafactor_plan_t* out) {
  if (!prm || !out || n < 1) return stk_fail(nullptr, STK_ERR_INVALID, "stk_adafactor_plan: NULL argument or no parameters");
  long long tiles = 0, line = 0, outs = 0, rm = 0, nb = 0;
  for (int j = 0; j < n; ++j) {
    stk_adafactor_param_t& d = prm[j];
    long long numel = 1;
    for (int k = 0; k < 4; ++k) {
      if (d.size[k] < 1) return stk_fail(nullptr, STK_ERR_INVALID, "stk_adafactor_plan: sizes must be >= 1");
      numel *= d.size[k];
    }
    if (numel != d.numel || numel >= (1ll << 31))
      return stk_fail(nullptr, STK_ERR_INVALID, "stk_adafactor_plan: numel must equal the product of the sizes and be < 2^31");
    // dense: the dims of size > 1, by decreasing stride, tile [0, numel) exactly
    long long expect = 1;
    int order[4] = {0, 1, 2, 3};
    for (int a = 0; a < 4; ++a)
      for (int b = a + 1; b < 4; ++b)
        if (d.stride[order[b]] < d.stride[order[a]]) std::swap(order[a], order[b]);
    for (int k = 0; k < 4; ++k) {
      const int dim = order[k];
      if (d.size[dim] == 1) continue;
      if (d.stride[dim] != expect) return stk_fail(nullptr, STK_ERR_INVALID, "stk_adafactor_plan: parameter is not dense");
      expect *= d.size[dim];
    }
    d.contiguous = (d.size[3] == 1 || d.stride[3] == 1) && (d.size[2] == 1 || d.stride[2] == d.size[3]) &&
                   (d.size[1] == 1 || d.stride[1] == d.size[2] * d.size[3]) &&
                   (d.size[0] == 1 || d.stride[0] == d.size[1] * d.size[2] * d.size[3]);
    d.tile0 = (int32_t)tiles;
    tiles += (numel + kAfTile - 1) / kAfTile;
    d.line0 = line;
    d.out0 = outs;
    d.b0 = (int32_t)nb;
    const long long B = (long long)d.size[0] * d.size[1], R = d.size[2], C = d.size[3];
    if (d.factored) {
      line += B * R * ((C + kAfChunk - 1) / kAfChunk) + B * C * ((R + kAfChunk - 1) / kAfChunk);
      outs += B * R + B * C;
      nb += B;
      if (R > 32) rm = (rm + 31) & ~31ll;
      d.rm0 = rm;
      rm += R > 32 ? 32 * B : B;
    } else {
      d.rm0 = rm;
    }
  }
  if (tiles >= (1ll << 31) || nb >= (1ll << 31)) return stk_fail(nullptr, STK_ERR_INVALID, "stk_adafactor_plan: too large");
  out->n_params = n;
  out->n_tiles = (int32_t)tiles;
  out->n_b = (int32_t)nb;
  out->pad_ = 0;
  out->n_line = line;
  out->n_out = outs;
  out->n_rm = rm;
  out->workspace_bytes = 2 * align16(tiles * 4) + align16(line * 4) + align16(nb * 4) + align16(n * sizeof(AfScal));
  return STK_OK;
}

int stk_adafactor_step(stk_ctx* c, const stk_adafactor_args_t* a, void* stream) {
  STK_REQUIRE(c, c && a && a->hyper && a->params && a->plan && a->param_group && a->steps && a->master && a->state &&
                     a->workspace && a->grad, "stk_adafactor_step: NULL argument");
  STK_REQUIRE(c, a->n_groups >= 1 && a->n_groups <= STK_MAX_GROUPS, "stk_adafactor_step: n_groups must be in [1, 8]");
  STK_REQUIRE(c, a->plan->n_params >= 1, "stk_adafactor_step: empty plan");
  STK_REQUIRE(c, (reinterpret_cast<uintptr_t>(a->workspace) & 15) == 0, "stk_adafactor_step: workspace must be 16-byte aligned");
  STK_REQUIRE(c, a->grad_raw ? (a->grad_dtype == STK_BF16 || a->grad_dtype == STK_F32) : a->grad_dtype == STK_F32,
              "stk_adafactor_step: gradients must be a bf16 / fp32 raw bucket or fp32 main gradients");
  STK_REQUIRE(c, a->lp == nullptr || a->lp_dtype == STK_BF16 || a->lp_dtype == STK_F32, "stk_adafactor_step: lp dtype");
  STK_REQUIRE(c, a->clip_kind >= STK_CLIP_NONE && a->clip_kind <= STK_CLIP_VALUE, "stk_adafactor_step: clip kind");
  std::lock_guard<std::mutex> lk(c->mu);
  DeviceGuard g(c->device);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const stk_adafactor_plan_t& pl = *a->plan;

  AfParams p{};
  p.prm = a->params;
  p.n_params = pl.n_params;
  p.pgroup = a->param_group;
  p.steps = a->steps;
  p.master = a->master;
  p.state = a->state;
  char* ws = static_cast<char*>(a->workspace);
  p.part_w = reinterpret_cast<float*>(ws);
  ws += align16(size_t(pl.n_tiles) * 4);
  p.part_u = reinterpret_cast<float*>(ws);
  ws += align16(size_t(pl.n_tiles) * 4);
  p.line = reinterpret_cast<float*>(ws);
  ws += align16(size_t(pl.n_line) * 4);
  p.rmean = reinterpret_cast<float*>(ws);
  ws += align16(size_t(pl.n_b) * 4);
  p.scal = reinterpret_cast<AfScal*>(ws);
  p.grad = a->grad;
  p.acc = a->grad_raw ? a->acc : nullptr;
  p.lp = a->lp;
  p.scaler = c->scaler_dev;
  p.grad_mul = (float)a->grad_mul;
  p.clip_max_norm = (float)a->clip_max_norm;
  p.clip_value = (float)a->clip_value;
  p.grad_dtype = a->grad_dtype;
  p.raw = a->grad_raw ? 1 : 0;
  p.lp_dtype = a->lp_dtype;
  p.clip_kind = a->clip_kind;
  p.n_tiles = pl.n_tiles;
  p.n_line = pl.n_line;
  p.n_out = pl.n_out;
  p.n_rm = pl.n_rm;
  p.n_groups = a->n_groups;
  for (int gi = 0; gi < a->n_groups; ++gi) {
    const stk_adafactor_hyper_t& h = a->hyper[gi];
    p.g[gi] = AfGroup{h.lr, h.beta2_decay, h.eps1, h.eps2, h.d, h.weight_decay, h.eps1_none, h.maximize};
  }
  auto blocks = [](long long n) { return (unsigned)std::max<long long>(1, (n + kAfThreads - 1) / kAfThreads); };
  const unsigned warps_grid = blocks(32ll * pl.n_params);
  ProfScope prof(c, 1, s);
  k_af_sumsq_w<<<pl.n_tiles, kAfThreads, 0, s>>>(p);
  k_af_prologue<<<warps_grid, kAfThreads, 0, s>>>(p);
  if (pl.n_line > 0) {
    k_af_lines<<<blocks(pl.n_line), kAfThreads, 0, s>>>(p);
    k_af_lines_finish<<<blocks(pl.n_out), kAfThreads, 0, s>>>(p);
    k_af_rowmean<<<blocks(pl.n_rm), kAfThreads, 0, s>>>(p);
  }
  k_af_unorm<<<pl.n_tiles, kAfThreads, 0, s>>>(p);
  k_af_coef<<<warps_grid, kAfThreads, 0, s>>>(p);
  k_af_apply<<<pl.n_tiles, kAfThreads, 0, s>>>(p);
  STK_CUDA(c, cudaGetLastError());
  return STK_OK;
}

}  // extern "C"
