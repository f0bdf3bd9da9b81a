// k2_optim8bit.cu -- fused step of the 8-bit optimizers of stoke_b200.optim: AdamW8bit / Adam8bit, Lion8bit and
// AdEMAMix8bit, whose moments are stored as 8-bit codes into 256-entry maps, block-wise scaled by an fp32 absmax per 256
// elements (Dettmers et al., "8-bit Optimizers via Block-wise Quantization", 2022).  AdamW keeps m (signed map) and v
// (unsigned map), Lion its one m (signed), AdEMAMix m1 and m2 (both signed) and nu (unsigned).  Parameters below the
// class's min_8bit_size keep fp32 state in a compact buffer and take the same update without quantization.  Two
// stream-ordered launches, no host involvement:
//
//   1 k_q8_prologue  one thread per parameter: the skip / found_inf verdict, the step count advance and the step's
//                    scalars for pass 2 (AdamW: lr c2 / c1 and eps c2; AdEMAMix: ademamix_scalars and beta3_t; Lion: none)
//   2 k_q8_step      one warp per 256-element block, 8 contiguous elements per lane: dequantize the state, the update,
//                    each state's new block absmax by a NaN-propagating warp shuffle, the nearest codes by a binary search
//                    over the maps in shared memory (laid out level by level, see q8_nearest), the fp32 master and the
//                    low-precision copy; zeroes the raw bucket
//
// HBM bytes per element, world-1 bf16 raw route: reads g 2, master 4, codes 1 per state; writes master 4, codes 1 per
// state, bf16 copy 2, bucket zeroing 2 (AdamW 18, Lion 16, AdEMAMix 20; the absmax and the per-block table add 8 B per
// 256 elements and state).
// Every op is one IEEE fp32 operation, in the order of the class's step (no contraction), so the kernel is bit-identical
// to the class on CUDA.  Nothing adds across threads and nothing uses an atomic: two identical runs are bit-identical.  A
// skipped parameter (bit 7 of its group byte) or a step with found_inf leaves codes, absmax, master and count as they are;
// the raw bucket is zeroed all the same.
#include "ademamix.cuh"
#include "k1_common.cuh"

namespace stk {

constexpr int kQ8Block = STK_Q8_BLOCK;   // elements per quantization block (one warp)
constexpr int kQ8Threads = 256;

enum Q8Kind { Q8_ADAMW, Q8_LION, Q8_ADEMAMIX };

struct Q8Group {      // per group, converted once on the host
  double beta1, beta2, lr, eps;         // the bias corrections and the step scalars are formed in double from these
  float b1, one_m_b1, b2, one_m_b2, decay;   // decay: fp32(1 - lr wd), applied only when has_wd
  int has_wd;
};
struct Q8GroupX {     // per group, what Lion and AdEMAMix need besides Q8Group
  stk_ademamix_hyper_t a;   // AdEMAMix: alpha, beta3 and the warm-ups
  float lr, eps, wd;        // fp32(lr), fp32(eps), fp32(weight_decay)
  int pad_;
};
struct Q8Scal {       // per parameter, written by pass 1 for pass 2
  float step_size;    // fp32(lr c2 / c1)
  float eps_c2;       // fp32(eps c2)
  int live;           // stepped this step
  int pad_;
};
struct Q8ScalA {      // AdEMAMix's, in the same workspace (32 bytes per parameter)
  float4 s;           // ademamix_scalars: fp32 {1 / bc1, 1 / sqrt(bc2), alpha_t, 1 - beta3_t}
  float beta3;        // fp32(beta3_t)
  int live;
  int pad_[2];
};

struct Q8Params {
  const stk_adam8bit_param_t* prm;
  const int32_t* block_param;
  int n_params, n_blocks;
  const uint8_t* pgroup;
  int32_t* steps;
  Q8Scal* scal;
  float* master;
  uint8_t* code1;
  uint8_t* code2;
  float* absmax1;
  float* absmax2;
  const float* qmap1;
  const float* qmap2;
  float* small;       // fp32 state1 at [0, n_small), state2 at [n_small, 2 n_small), state3 at [2 n_small, 3 n_small)
  size_t n_small;
  const void* grad;
  const float* acc;
  void* lp;
  const stk_scaler_state_t* scaler;
  float grad_mul, clip_max_norm, clip_value;
  int raw, lp_dtype, clip_kind;
  Q8Group g[STK_MAX_GROUPS];
  // Lion and AdEMAMix only; after the fields above, so that AdamW's parameter offsets are those it always had
  uint8_t* code3;     // AdEMAMix's m2 (signed map)
  float* absmax3;
  Q8GroupX gx[STK_MAX_GROUPS];
};

__device__ __forceinline__ uint2 ld_stream8(const void* p) {
  uint2 v;
  asm volatile("ld.global.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p));
  return v;
}
__device__ __forceinline__ void st_stream8(void* p, const uint2& v) {
  asm volatile("st.global.L1::no_allocate.v2.u32 [%0], {%1,%2};" ::"l"(p), "r"(v.x), "r"(v.y) : "memory");
}
__device__ __forceinline__ uint32_t byte_of(const uint2& v, int e) { return ((e < 4 ? v.x : v.y) >> (8 * (e & 3))) & 0xffu; }

// The search tree of a sorted 256-entry map q, level by level: level k (0..7) holds the 2^k entries its k-th comparison
// can read, q[i 2^(8-k) + 2^(7-k) - 1] for i < 2^k, at tree[2^k - 1 + i].  In the sorted layout the candidates of the
// first levels are 32 or more entries apart and all fall in one shared-memory bank; here a level's candidates are
// adjacent, so levels 0-5 read without bank conflicts.
__device__ __forceinline__ float q8_tree_entry(const float* q, int idx) {
  const int k = 31 - __clz(idx + 1), i = idx + 1 - (1 << k);
  return q[i * (kQ8Block >> k) + (kQ8Block >> (k + 1)) - 1];
}

// The index of the map entry nearest to n: distances are fp32 subtractions |n - q[i]|, equal distances go to the lower
// index, and a NaN n takes the code of 0.  n is first clamped into [q[0], q[255]] (lo and hi arrive as those two), so
// an n above the map -- +inf from an overflowing 1 / absmax, or 1.0 under a checkpoint's map that tops out below 1 --
// takes code 255 and one below it code 0, even where the two top (bottom) entries are equally far from n in fp32.
// Eight comparisons down the tree give P, the number of entries among q[0..254] below n (the branchless lower bound);
// the last entry found below n is q[P - 1] and the last found at or above it q[P] (q[255] when P = 255), so the nearest
// is one of the two without reading the map again.
__device__ __forceinline__ uint32_t q8_nearest(const float* tree, float lo, float hi, float n) {
  if (n != n) n = 0.f;
  n = fminf(fmaxf(n, lo), hi);
  int node = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const float t = tree[node];
    const bool lt = t < n;
    lo = lt ? t : lo;
    hi = lt ? hi : t;
    node = 2 * node + (lt ? 2 : 1);
  }
  const int P = node - (kQ8Block - 1);
  const float dl = fabsf(__fsub_rn(n, lo)), dh = fabsf(__fsub_rn(n, hi));
  return (P > 0 && dl <= dh) ? (uint32_t)(P - 1) : (uint32_t)P;
}

// the codes of 8 elements (x already multiplied by the block's 1 / absmax); elements at or after `valid` keep `old`'s
// bytes.  q: the sorted map (its first and last entries seed the search), tree: its level-by-level layout
__device__ __forceinline__ uint2 q8_encode(const float* tree, const float* q, const float (&x)[8], int valid,
                                           const uint2& old) {
  const float q0 = q[0], q255 = q[kQ8Block - 1];
  uint32_t b[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) b[e] = e < valid ? q8_nearest(tree, q0, q255, x[e]) : byte_of(old, e);
  return make_uint2(b[0] | (b[1] << 8) | (b[2] << 16) | (b[3] << 24), b[4] | (b[5] << 8) | (b[6] << 16) | (b[7] << 24));
}

// torch's where(absmax == 0, 0, absmax.reciprocal()): a correctly rounded reciprocal, NaN for a NaN absmax, 0 for inf
__device__ __forceinline__ float q8_inv(float absmax) { return absmax == 0.f ? 0.f : __frcp_rn(absmax); }

// ---- 1: per-parameter verdict, step count, step scalars ----------------------------------------------------------------
template <int KIND>
__global__ void __launch_bounds__(kQ8Threads) k_q8_prologue(const Q8Params p) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= p.n_params) return;
  const unsigned gb = p.pgroup[j];
  const Q8Group& h = p.g[gb & 0x7f];
  if constexpr (KIND == Q8_ADEMAMIX) {
    Q8ScalA o{};
    if (p.scaler->found_inf == 0 && !(gb & 0x80u)) {
      const int32_t t = p.steps[j] + 1;
      o.s = ademamix_scalars(h.beta1, h.beta2, p.gx[gb & 0x7f].a, (double)t, &o.beta3);
      o.live = 1;
      p.steps[j] = t;
    }
    reinterpret_cast<Q8ScalA*>(p.scal)[j] = o;
  } else {
    Q8Scal o{0.f, 0.f, 0, 0};
    if (p.scaler->found_inf == 0 && !(gb & 0x80u)) {
      const int32_t t = p.steps[j] + 1;
      if constexpr (KIND == Q8_ADAMW) {
        // c1 = 1 - beta1 ** t, c2 = sqrt(1 - beta2 ** t), python doubles
        const double c1 = 1.0 - pow(h.beta1, (double)t), c2 = sqrt(1.0 - pow(h.beta2, (double)t));
        o.step_size = (float)(h.lr * c2 / c1);
        o.eps_c2 = (float)(h.eps * c2);
      }
      o.live = 1;
      p.steps[j] = t;
    }
    p.scal[j] = o;
  }
}

// ---- 2: the update ------------------------------------------------------------------------------------------------------
template <int KIND>
struct Q8Traits {
  using Scal = Q8Scal;
  static constexpr int kMaps = 2;   // the signed map (s_q[0]) and the unsigned one (s_q[1])
};
template <>
struct Q8Traits<Q8_LION> {
  using Scal = Q8Scal;
  static constexpr int kMaps = 1;   // Lion's m: the signed map only
};
template <>
struct Q8Traits<Q8_ADEMAMIX> {
  using Scal = Q8ScalA;
  static constexpr int kMaps = 2;
};

template <int KIND, int GDT>
__global__ void __launch_bounds__(kQ8Threads) k_q8_step(const Q8Params p) {
  constexpr int kMaps = Q8Traits<KIND>::kMaps;
  constexpr bool kV = KIND != Q8_LION;         // a second state on the unsigned map (AdamW's v, AdEMAMix's nu)
  constexpr bool kM3 = KIND == Q8_ADEMAMIX;    // a third state on the signed map (AdEMAMix's m2)
  __shared__ float s_q[kMaps][kQ8Block];      // the maps, sorted (dequantization)
  __shared__ float s_tree[kMaps][kQ8Block];   // their search trees (255 entries each)
  for (int i = threadIdx.x; i < kMaps * kQ8Block; i += kQ8Threads) {
    const float* q = i < kQ8Block ? p.qmap1 : p.qmap2;
    const int j = i % kQ8Block;
    s_q[i / kQ8Block][j] = q[j];
    if (j < kQ8Block - 1) s_tree[i / kQ8Block][j] = q8_tree_entry(q, j);
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const float inv_scale = p.raw ? (float)(1.0 / (double)p.scaler->scale) : 1.f;
  const float coef = clip_coef(p.clip_kind, p.clip_max_norm, p.scaler);
  const int warps = gridDim.x * (kQ8Threads / 32);
  for (int b = blockIdx.x * (kQ8Threads / 32) + (threadIdx.x >> 5); b < p.n_blocks; b += warps) {
    const int j = p.block_param[b];
    const stk_adam8bit_param_t d = p.prm[j];
    const typename Q8Traits<KIND>::Scal sc = reinterpret_cast<const typename Q8Traits<KIND>::Scal*>(p.scal)[j];
    const int q0 = (b - d.block0) * kQ8Block;
    const int valid = min(8, d.numel - q0 - 8 * lane);   // <= 0: this lane is past the parameter's end
    const size_t e0 = d.offset + (size_t)q0 + 8 * lane;  // first flat element of this lane
    const size_t vi = e0 >> 3;
    if (!sc.live) {   // skipped: the bucket is consumed all the same
      if (p.raw && valid > 0) InVec<GDT>::zero(const_cast<void*>(p.grad), vi);
      continue;       // uniform per warp
    }
    const Q8Group& h = p.g[p.pgroup[j] & 0x7f];
    const bool quant = d.small < 0;
    float g[8], w[8], m[8], v[8], m3[8];
    uint2 c1 = make_uint2(0, 0), c2 = make_uint2(0, 0), c3 = make_uint2(0, 0);
    if (valid > 0) {
      InVec<GDT>::load(p.grad, vi, g);
      if (p.acc != nullptr) {
        float a[8];
        InVec<STK_F32>::load(p.acc, vi, a);
#pragma unroll
        for (int e = 0; e < 8; ++e) g[e] += a[e];
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) g[e] = form_grad(g[e], p.raw != 0, p.grad_mul, inv_scale, p.clip_kind, coef, p.clip_value);
      InVec<STK_F32>::load(p.master, vi, w);
      if (quant) {
        c1 = ld_stream8(p.code1 + e0);
        if constexpr (kV) c2 = ld_stream8(p.code2 + e0);
        if constexpr (kM3) c3 = ld_stream8(p.code3 + e0);
        const float a1 = p.absmax1[b];
        const float a2 = kV ? p.absmax2[b] : 0.f;
        const float a3 = kM3 ? p.absmax3[b] : 0.f;
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          m[e] = __fmul_rn(s_q[0][byte_of(c1, e)], a1);   // deq(code) = qmap[code] * absmax
          if constexpr (kV) v[e] = __fmul_rn(s_q[kMaps - 1][byte_of(c2, e)], a2);
          if constexpr (kM3) m3[e] = __fmul_rn(s_q[0][byte_of(c3, e)], a3);
        }
      } else {
        const size_t si = ((size_t)d.small + q0 + 8 * lane) >> 3;
        InVec<STK_F32>::load(p.small, si, m);
        if constexpr (kV) InVec<STK_F32>::load(p.small + p.n_small, si, v);
        if constexpr (kM3) InVec<STK_F32>::load(p.small + 2 * p.n_small, si, m3);
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        if (e >= valid) continue;   // the parameter's last vector may end in padding: left as it is
        const float gg = g[e];
        if constexpr (KIND == Q8_ADAMW) {
          m[e] = __fadd_rn(__fmul_rn(m[e], h.b1), __fmul_rn(gg, h.one_m_b1));                  // m * b1 + g * (1 - b1)
          v[e] = __fadd_rn(__fmul_rn(v[e], h.b2), __fmul_rn(__fmul_rn(gg, gg), h.one_m_b2));   // v * b2 + (g * g) * (1 - b2)
          float ww = w[e];
          if (h.has_wd) ww = __fmul_rn(ww, h.decay);                                            // w * (1 - lr wd)
          const float den = __fadd_rn(__fsqrt_rn(v[e]), sc.eps_c2);                             // sqrt(v) + eps c2
          w[e] = __fsub_rn(ww, __fmul_rn(__fdiv_rn(m[e], den), sc.step_size));                  // w - (m / den) * step
        } else if constexpr (KIND == Q8_LION) {
          const Q8GroupX& x = p.gx[p.pgroup[j] & 0x7f];
          float ww = w[e];
          if (h.has_wd) ww = __fmul_rn(ww, h.decay);                                            // w * (1 - lr wd)
          const float c = __fadd_rn(__fmul_rn(m[e], h.b1), __fmul_rn(gg, h.one_m_b1));         // m * b1 + g * (1 - b1)
          const float s = (float)((c > 0.f) - (c < 0.f));                                       // sign: NaN, +-0 give 0
          w[e] = __fsub_rn(ww, __fmul_rn(s, x.lr));                                             // w - s * lr
          m[e] = __fadd_rn(__fmul_rn(m[e], h.b2), __fmul_rn(gg, h.one_m_b2));                  // m * b2 + g * (1 - b2)
        } else {
          const Q8GroupX& x = p.gx[p.pgroup[j] & 0x7f];
          m[e] = __fadd_rn(__fmul_rn(m[e], h.b1), __fmul_rn(gg, h.one_m_b1));                  // m1 * b1 + g * (1 - b1)
          m3[e] = __fadd_rn(__fmul_rn(m3[e], sc.beta3), __fmul_rn(gg, sc.s.w));                // m2 * b3_t + g * (1 - b3_t)
          v[e] = __fadd_rn(__fmul_rn(v[e], h.b2), __fmul_rn(__fmul_rn(gg, gg), h.one_m_b2));   // nu * b2 + (g * g) * (1 - b2)
          const float den = __fadd_rn(__fmul_rn(__fsqrt_rn(v[e]), sc.s.y), x.eps);             // sqrt(nu) / sqrt(bc2) + eps
          float u = __fdiv_rn(__fadd_rn(__fmul_rn(m[e], sc.s.x), __fmul_rn(m3[e], sc.s.z)), den);   // (m1 / bc1 + m2 a_t) / den
          if (h.has_wd) u = __fadd_rn(u, __fmul_rn(w[e], x.wd));                               // u + w * wd
          w[e] = __fsub_rn(w[e], __fmul_rn(u, x.lr));                                           // w - u * lr
        }
      }
    }
    if (quant) {      // uniform per warp: every lane takes part in the shuffles
      float x1 = 0.f, x2 = 0.f, x3 = 0.f;
#pragma unroll
      for (int e = 0; e < 8; ++e)
        if (e < valid) {
          x1 = fmax_nan(x1, fabsf(m[e]));
          if constexpr (kV) x2 = fmax_nan(x2, fabsf(v[e]));
          if constexpr (kM3) x3 = fmax_nan(x3, fabsf(m3[e]));
        }
      const float a1 = warp_reduce<true>(x1);
      const float a2 = kV ? warp_reduce<true>(x2) : 0.f;
      const float a3 = kM3 ? warp_reduce<true>(x3) : 0.f;
      if (valid > 0) {
        const float i1 = q8_inv(a1), i2 = q8_inv(a2), i3 = q8_inv(a3);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          m[e] = __fmul_rn(m[e], i1);
          if constexpr (kV) v[e] = __fmul_rn(v[e], i2);
          if constexpr (kM3) m3[e] = __fmul_rn(m3[e], i3);
        }
        st_stream8(p.code1 + e0, q8_encode(s_tree[0], s_q[0], m, valid, c1));
        if constexpr (kV) st_stream8(p.code2 + e0, q8_encode(s_tree[kMaps - 1], s_q[kMaps - 1], v, valid, c2));
        if constexpr (kM3) st_stream8(p.code3 + e0, q8_encode(s_tree[0], s_q[0], m3, valid, c3));
      }
      if (lane == 0) {
        p.absmax1[b] = a1;
        if constexpr (kV) p.absmax2[b] = a2;
        if constexpr (kM3) p.absmax3[b] = a3;
      }
    } else if (valid > 0) {
      const size_t si = ((size_t)d.small + q0 + 8 * lane) >> 3;
      st_stream_f8(p.small + si * 8, m);
      if constexpr (kV) st_stream_f8(p.small + p.n_small + si * 8, v);
      if constexpr (kM3) st_stream_f8(p.small + 2 * p.n_small + si * 8, m3);
    }
    if (valid > 0) {
      st_stream_f8(p.master + vi * 8, w);
      if (p.lp != nullptr) {
        if (p.lp_dtype == STK_BF16) store_out<STK_BF16>(p.lp, vi, w);
        else store_out<STK_F32>(p.lp, vi, w);
      }
      if (p.raw) InVec<GDT>::zero(const_cast<void*>(p.grad), vi);
    }
  }
}

template <int KIND, int GDT>
void q8_launch(const Q8Params& p, int sm_count, cudaStream_t s) {
  k_q8_prologue<KIND><<<(p.n_params + kQ8Threads - 1) / kQ8Threads, kQ8Threads, 0, s>>>(p);
  const int per_cta = kQ8Threads / 32;
  const int grid = (int)std::min<long long>((p.n_blocks + per_cta - 1) / per_cta, 16ll * sm_count);
  k_q8_step<KIND, GDT><<<std::max(grid, 1), kQ8Threads, 0, s>>>(p);
}

// The checks every 8-bit entry point shares, and the parameters they fill in from stk_adam8bit_args_t.  `states`: 1
// (Lion: code1 / absmax1 / qmap1), 2 (AdamW: also code2 / absmax2 / qmap2) or 3 (AdEMAMix: also code3 / absmax3).
int q8_check(stk_ctx* c, const stk_adam8bit_args_t* a, int states, const uint8_t* code3, const float* absmax3,
             const char* fn) {
  auto fail = [&](const char* what) { return stk_fail(c, STK_ERR_INVALID, std::string(fn) + ": " + what); };
  if (!(c && a && a->hyper && a->params && a->block_param && a->param_group && a->steps && a->master && a->workspace &&
        a->grad && a->qmap1 && (states < 2 || a->qmap2)))
    return fail("NULL argument");
  if (!(a->n_groups >= 1 && a->n_groups <= STK_MAX_GROUPS)) return fail("n_groups must be in [1, 8]");
  if (!(a->n_params >= 1 && a->n_blocks >= 1)) return fail("no parameters");
  if (reinterpret_cast<uintptr_t>(a->workspace) & 15) return fail("workspace must be 16-byte aligned");
  if (!(a->grad_raw ? (a->grad_dtype == STK_BF16 || a->grad_dtype == STK_F32) : a->grad_dtype == STK_F32))
    return fail("gradients must be a bf16 / fp32 raw bucket or fp32 main gradients");
  if (!(a->lp == nullptr || a->lp_dtype == STK_BF16 || a->lp_dtype == STK_F32)) return fail("lp dtype");
  if (!(a->clip_kind >= STK_CLIP_NONE && a->clip_kind <= STK_CLIP_VALUE)) return fail("clip kind");
  if (!((a->code1 && a->absmax1 && (states < 2 || (a->code2 && a->absmax2)) && (states < 3 || (code3 && absmax3))) ||
        a->n_small > 0))
    return fail(states == 1 ? "the 8-bit parameters need code1 and absmax1"
                : states == 2 ? "the 8-bit parameters need code1, code2, absmax1 and absmax2"
                              : "the 8-bit parameters need code1, code2, code3, absmax1, absmax2 and absmax3");
  if (!(a->n_small == 0 || (a->small && a->n_small % 8 == 0)))
    return fail("the small parameters need `small`, n_small a multiple of 8");
  return STK_OK;
}

void q8_fill(stk_ctx* c, const stk_adam8bit_args_t* a, Q8Params& p) {
  p.prm = a->params;
  p.block_param = a->block_param;
  p.n_params = a->n_params;
  p.n_blocks = a->n_blocks;
  p.pgroup = a->param_group;
  p.steps = a->steps;
  p.scal = reinterpret_cast<Q8Scal*>(a->workspace);
  p.master = a->master;
  p.code1 = a->code1;
  p.code2 = a->code2;
  p.absmax1 = a->absmax1;
  p.absmax2 = a->absmax2;
  p.qmap1 = a->qmap1;
  p.qmap2 = a->qmap2;
  p.small = a->small;
  p.n_small = a->n_small;
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
  for (int gi = 0; gi < a->n_groups; ++gi) {
    const stk_adam8bit_hyper_t& h = a->hyper[gi];
    Q8Group& o = p.g[gi];
    o.beta1 = h.beta1;
    o.beta2 = h.beta2;
    o.lr = h.lr;
    o.eps = h.eps;
    o.b1 = (float)h.beta1;
    o.one_m_b1 = (float)(1.0 - h.beta1);
    o.b2 = (float)h.beta2;
    o.one_m_b2 = (float)(1.0 - h.beta2);
    o.decay = (float)(1.0 - h.lr * h.weight_decay);
    o.has_wd = h.weight_decay != 0.0;
    Q8GroupX& x = p.gx[gi];
    x.lr = (float)h.lr;
    x.eps = (float)h.eps;
    x.wd = (float)h.weight_decay;
  }
}

template <int KIND>
int q8_run(stk_ctx* c, const stk_adam8bit_args_t* a, const Q8Params& p, void* stream) {
  std::lock_guard<std::mutex> lk(c->mu);
  DeviceGuard g(c->device);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const bool bf16 = a->grad_raw && a->grad_dtype == STK_BF16;
  ProfScope prof(c, 1, s);
  if (bf16) q8_launch<KIND, STK_BF16>(p, c->sm_count, s);
  else q8_launch<KIND, STK_F32>(p, c->sm_count, s);
  STK_CUDA(c, cudaGetLastError());
  return STK_OK;
}

}  // namespace stk

using namespace stk;

extern "C" {

int stk_adam8bit_step(stk_ctx* c, const stk_adam8bit_args_t* a, void* stream) {
  if (int rc = q8_check(c, a, 2, nullptr, nullptr, "stk_adam8bit_step")) return rc;
  Q8Params p{};
  q8_fill(c, a, p);
  return q8_run<Q8_ADAMW>(c, a, p, stream);
}

int stk_lion8bit_step(stk_ctx* c, const stk_adam8bit_args_t* a, void* stream) {
  if (int rc = q8_check(c, a, 1, nullptr, nullptr, "stk_lion8bit_step")) return rc;
  Q8Params p{};
  q8_fill(c, a, p);
  return q8_run<Q8_LION>(c, a, p, stream);
}

int stk_ademamix8bit_step(stk_ctx* c, const stk_adam8bit_args_t* a, const stk_ademamix_hyper_t* ademamix, uint8_t* code3,
                          float* absmax3, void* stream) {
  if (int rc = q8_check(c, a, 3, code3, absmax3, "stk_ademamix8bit_step")) return rc;
  if (!ademamix) return stk_fail(c, STK_ERR_INVALID, "stk_ademamix8bit_step: NULL argument");
  Q8Params p{};
  q8_fill(c, a, p);
  p.code3 = code3;
  p.absmax3 = absmax3;
  for (int gi = 0; gi < a->n_groups; ++gi) p.gx[gi].a = ademamix[gi];
  return q8_run<Q8_ADEMAMIX>(c, a, p, stream);
}

}  // extern "C"
