// k2_optim8bit.cu -- fused step of stoke_b200.optim.AdamW8bit / Adam8bit: AdamW with its two moments stored as 8-bit
// codes into two 256-entry maps, block-wise scaled by an fp32 absmax per 256 elements (Dettmers et al., "8-bit Optimizers
// via Block-wise Quantization", 2022).  Parameters below the class's min_8bit_size keep fp32 moments in a compact buffer
// and take the same update without quantization.  Two stream-ordered launches, no host involvement:
//
//   1 k_q8_prologue  one thread per parameter: the skip / found_inf verdict, the step count advance and the step's
//                    scalars (lr c2 / c1 and eps c2 from python-double formulas) for pass 2
//   2 k_q8_step      one warp per 256-element block, 8 contiguous elements per lane: dequantize m and v, the update,
//                    the block's new absmax by a NaN-propagating warp shuffle, the nearest codes by a binary search over
//                    the maps in shared memory (laid out level by level, see q8_nearest), the fp32 master and the
//                    low-precision copy; zeroes the raw bucket
//
// HBM bytes per element, world-1 bf16 raw route: reads g 2, master 4, codes 2; writes master 4, codes 2, bf16 copy 2,
// bucket zeroing 2 (18; the absmax and the per-block table add 12 B per 256 elements).
// Every op is one IEEE fp32 operation, in the order of AdamW8bit.step (no contraction), so the kernel is bit-identical to
// the class on CUDA.  Nothing adds across threads and nothing uses an atomic: two identical runs are bit-identical.  A
// skipped parameter (bit 7 of its group byte) or a step with found_inf leaves codes, absmax, master and count as they are;
// the raw bucket is zeroed all the same.
#include "k1_common.cuh"

namespace stk {

constexpr int kQ8Block = STK_Q8_BLOCK;   // elements per quantization block (one warp)
constexpr int kQ8Threads = 256;

struct Q8Group {      // per group, converted once on the host
  double beta1, beta2, lr, eps;         // the bias corrections and the step scalars are formed in double from these
  float b1, one_m_b1, b2, one_m_b2, decay;   // decay: fp32(1 - lr wd), applied only when has_wd
  int has_wd;
};
struct Q8Scal {       // per parameter, written by pass 1 for pass 2
  float step_size;    // fp32(lr c2 / c1)
  float eps_c2;       // fp32(eps c2)
  int live;           // stepped this step
  int pad_;
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
  float* small;       // fp32 state1 at [0, n_small), state2 at [n_small, 2 n_small)
  size_t n_small;
  const void* grad;
  const float* acc;
  void* lp;
  const stk_scaler_state_t* scaler;
  float grad_mul, clip_max_norm, clip_value;
  int raw, lp_dtype, clip_kind;
  Q8Group g[STK_MAX_GROUPS];
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
__global__ void __launch_bounds__(kQ8Threads) k_q8_prologue(const Q8Params p) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= p.n_params) return;
  const unsigned gb = p.pgroup[j];
  const Q8Group& h = p.g[gb & 0x7f];
  Q8Scal o{0.f, 0.f, 0, 0};
  if (p.scaler->found_inf == 0 && !(gb & 0x80u)) {
    const int32_t t = p.steps[j] + 1;
    // c1 = 1 - beta1 ** t, c2 = sqrt(1 - beta2 ** t), python doubles
    const double c1 = 1.0 - pow(h.beta1, (double)t), c2 = sqrt(1.0 - pow(h.beta2, (double)t));
    o.step_size = (float)(h.lr * c2 / c1);
    o.eps_c2 = (float)(h.eps * c2);
    o.live = 1;
    p.steps[j] = t;
  }
  p.scal[j] = o;
}

// ---- 2: the update ------------------------------------------------------------------------------------------------------
template <int GDT>
__global__ void __launch_bounds__(kQ8Threads) k_q8_step(const Q8Params p) {
  __shared__ float s_q[2][kQ8Block];      // the maps, sorted (dequantization)
  __shared__ float s_tree[2][kQ8Block];   // their search trees (255 entries each)
  for (int i = threadIdx.x; i < 2 * kQ8Block; i += kQ8Threads) {
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
    const Q8Scal sc = p.scal[j];
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
    float g[8], w[8], m[8], v[8];
    uint2 c1 = make_uint2(0, 0), c2 = make_uint2(0, 0);
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
        c2 = ld_stream8(p.code2 + e0);
        const float a1 = p.absmax1[b], a2 = p.absmax2[b];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          m[e] = __fmul_rn(s_q[0][byte_of(c1, e)], a1);   // deq(code) = qmap[code] * absmax
          v[e] = __fmul_rn(s_q[1][byte_of(c2, e)], a2);
        }
      } else {
        const size_t si = ((size_t)d.small + q0 + 8 * lane) >> 3;
        InVec<STK_F32>::load(p.small, si, m);
        InVec<STK_F32>::load(p.small + p.n_small, si, v);
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        if (e >= valid) continue;   // the parameter's last vector may end in padding: left as it is
        const float gg = g[e];
        m[e] = __fadd_rn(__fmul_rn(m[e], h.b1), __fmul_rn(gg, h.one_m_b1));                  // m * b1 + g * (1 - b1)
        v[e] = __fadd_rn(__fmul_rn(v[e], h.b2), __fmul_rn(__fmul_rn(gg, gg), h.one_m_b2));   // v * b2 + (g * g) * (1 - b2)
        float ww = w[e];
        if (h.has_wd) ww = __fmul_rn(ww, h.decay);                                            // w * (1 - lr wd)
        const float den = __fadd_rn(__fsqrt_rn(v[e]), sc.eps_c2);                             // sqrt(v) + eps c2
        w[e] = __fsub_rn(ww, __fmul_rn(__fdiv_rn(m[e], den), sc.step_size));                  // w - (m / den) * step
      }
    }
    if (quant) {      // uniform per warp: every lane takes part in the shuffles
      float x1 = 0.f, x2 = 0.f;
#pragma unroll
      for (int e = 0; e < 8; ++e)
        if (e < valid) {
          x1 = fmax_nan(x1, fabsf(m[e]));
          x2 = fmax_nan(x2, fabsf(v[e]));
        }
      const float a1 = warp_reduce<true>(x1), a2 = warp_reduce<true>(x2);
      if (valid > 0) {
        const float i1 = q8_inv(a1), i2 = q8_inv(a2);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          m[e] = __fmul_rn(m[e], i1);
          v[e] = __fmul_rn(v[e], i2);
        }
        st_stream8(p.code1 + e0, q8_encode(s_tree[0], s_q[0], m, valid, c1));
        st_stream8(p.code2 + e0, q8_encode(s_tree[1], s_q[1], v, valid, c2));
      }
      if (lane == 0) {
        p.absmax1[b] = a1;
        p.absmax2[b] = a2;
      }
    } else if (valid > 0) {
      const size_t si = ((size_t)d.small + q0 + 8 * lane) >> 3;
      st_stream_f8(p.small + si * 8, m);
      st_stream_f8(p.small + p.n_small + si * 8, v);
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

template <int GDT>
void q8_launch(const Q8Params& p, int sm_count, cudaStream_t s) {
  k_q8_prologue<<<(p.n_params + kQ8Threads - 1) / kQ8Threads, kQ8Threads, 0, s>>>(p);
  const int per_cta = kQ8Threads / 32;
  const int grid = (int)std::min<long long>((p.n_blocks + per_cta - 1) / per_cta, 16ll * sm_count);
  k_q8_step<GDT><<<std::max(grid, 1), kQ8Threads, 0, s>>>(p);
}

}  // namespace stk

using namespace stk;

extern "C" {

int stk_adam8bit_step(stk_ctx* c, const stk_adam8bit_args_t* a, void* stream) {
  STK_REQUIRE(c, c && a && a->hyper && a->params && a->block_param && a->param_group && a->steps && a->master &&
                     a->workspace && a->grad && a->qmap1 && a->qmap2,
              "stk_adam8bit_step: NULL argument");
  STK_REQUIRE(c, a->n_groups >= 1 && a->n_groups <= STK_MAX_GROUPS, "stk_adam8bit_step: n_groups must be in [1, 8]");
  STK_REQUIRE(c, a->n_params >= 1 && a->n_blocks >= 1, "stk_adam8bit_step: no parameters");
  STK_REQUIRE(c, (reinterpret_cast<uintptr_t>(a->workspace) & 15) == 0, "stk_adam8bit_step: workspace must be 16-byte aligned");
  STK_REQUIRE(c, a->grad_raw ? (a->grad_dtype == STK_BF16 || a->grad_dtype == STK_F32) : a->grad_dtype == STK_F32,
              "stk_adam8bit_step: gradients must be a bf16 / fp32 raw bucket or fp32 main gradients");
  STK_REQUIRE(c, a->lp == nullptr || a->lp_dtype == STK_BF16 || a->lp_dtype == STK_F32, "stk_adam8bit_step: lp dtype");
  STK_REQUIRE(c, a->clip_kind >= STK_CLIP_NONE && a->clip_kind <= STK_CLIP_VALUE, "stk_adam8bit_step: clip kind");
  STK_REQUIRE(c, (a->code1 && a->code2 && a->absmax1 && a->absmax2) || a->n_small > 0,
              "stk_adam8bit_step: the 8-bit parameters need code1, code2, absmax1 and absmax2");
  STK_REQUIRE(c, a->n_small == 0 || (a->small && a->n_small % 8 == 0),
              "stk_adam8bit_step: the small parameters need `small`, n_small a multiple of 8");
  std::lock_guard<std::mutex> lk(c->mu);
  DeviceGuard g(c->device);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);

  Q8Params p{};
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
  }
  const bool bf16 = a->grad_raw && a->grad_dtype == STK_BF16;
  ProfScope prof(c, 1, s);
  if (bf16) q8_launch<STK_BF16>(p, c->sm_count, s);
  else q8_launch<STK_F32>(p, c->sm_count, s);
  STK_CUDA(c, cudaGetLastError());
  return STK_OK;
}

}  // extern "C"
