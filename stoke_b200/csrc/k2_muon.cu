// k2_muon.cu -- fused Muon step (torch.optim.Muon and the Muon half of stoke_b200.optim.MuonWithAuxAdamW): momentum,
// Newton-Schulz orthogonalisation on bf16 tensor cores, batched over every matrix of the step, and the update.  Stream-
// ordered launches, no host involvement:
//
//   1 k_mu_prep       tile pass over each matrix's elements (kMuTile per block): g, buf = lerp(buf, g, 1 - momentum),
//                     u, X = bf16(u) (transposed when the parameter has more rows than columns), per-tile sum of X^2;
//                     writes buf and X, zeroes the raw bucket
//   2 k_mu_fold       one warp per matrix: folds its tile partials in index order into n = bf16(||X||), clamped at eps;
//                     advances the step count
//   3 k_mu_scale      tile pass over X: X = bf16(X / n)
//   4 k_mu_gemm       3 launches per Newton-Schulz step, each over every matrix still iterating: A = X X^T,
//                     B = b A + c A A (lower tile triangles, mirrored), X' = a X + B X (all tiles); 64 x 64 output tiles
//                     of mma.sync m16n8k16 bf16 with fp32 accumulation, the fp32 epilogue rounded once to bf16
//   5 k_mu_apply      tile pass: w = w (1 - lr wd) + (-lr ratio) X, the fp32 master and the low-precision copy
//
// Every sum adds in an order fixed by the shapes and these launch shapes only, and nothing uses a floating-point atomic:
// two identical runs are bit-identical.  A skipped matrix (bit 7 of its group byte) or a step with found_inf leaves
// master, buf and step count as they are; the raw bucket is zeroed all the same.
#include <cuda_bf16.h>

#include "k1_common.cuh"

namespace stk {

constexpr int kMuTile = STK_MUON_TILE;
constexpr int kMuThreads = 256;
constexpr int kMm = STK_MUON_MMA_TILE;  // output tile rows / columns
constexpr int kMk = 32;                 // k per shared-memory stage
constexpr int kMmThreads = 128;         // 2 x 2 warps of 32 x 32 outputs
constexpr int kLds = kMk + 8;           // shared row stride in bf16: 80 B, conflict-free fragment loads

typedef __nv_bfloat16 bf16;

struct MuGroup {      // per group, converted once on the host
  double lr;
  float one_m_mom, mom, keep, a, b, c, eps;   // keep = fp32(1 - lr wd); eps: bf16(eps) as a float
  int nesterov, ns_steps;
};
struct MuScal {       // per matrix, written by pass 2
  float n;            // bf16(||X||) clamped at eps
  int flags;          // bit 0: stepped this step
};

struct MuParams {
  const stk_muon_param_t* prm;
  int n_params;
  const uint8_t* pgroup;
  int32_t* steps;
  float* master;
  float* buf;
  bf16* x0;
  bf16* x1;
  bf16* a;
  bf16* b;
  MuScal* scal;
  float* part;        // per tile: sum of X^2
  const void* grad;
  const float* acc;
  void* lp;
  const stk_scaler_state_t* scaler;
  float grad_mul, clip_max_norm, clip_value;
  int raw, lp_dtype, clip_kind, max_ns;
  MuGroup g[STK_MAX_GROUPS];
};

// largest j with key(prm[j]) <= t: the matrix owning tile t (a matrix without tiles shares its first tile with the
// next one, which then wins)
template <int KEY>
__device__ __forceinline__ int mu_find(const MuParams& p, int t) {
  int lo = 0, hi = p.n_params - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    const stk_muon_param_t& d = p.prm[mid];
    const int k = KEY == 0 ? d.tile0 : KEY == 1 ? d.tri0 : d.full0;
    if (k <= t) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ bool mu_live(const MuParams& p, unsigned gb) {
  return p.scaler->found_inf == 0 && !(gb & 0x80u);
}

// the element of X that holds flat element q of the parameter (row-major R x C; X is C x R when transposed)
__device__ __forceinline__ size_t mu_xi(const stk_muon_param_t& d, int64_t q) {
  if (!d.transposed) return (size_t)q;
  const int64_t C = d.rows, R = d.cols;   // the parameter's shape: R x C with R > C
  return (size_t)((q % C) * R + q / C);
}

// ---- 1: momentum, X, partial sums ------------------------------------------------------------------------------------
template <int GDT>
__global__ void __launch_bounds__(kMuThreads) k_mu_prep(const MuParams p) {
  __shared__ float s_red[32];
  const int tile = blockIdx.x;
  const stk_muon_param_t d = p.prm[mu_find<0>(p, tile)];
  const unsigned gb = p.pgroup[d.param];
  const MuGroup& h = p.g[gb & 0x7f];
  const int64_t q0 = (int64_t)(tile - d.tile0) * kMuTile;
  const int nq = (int)min((int64_t)kMuTile, (int64_t)d.rows * d.cols - q0);
  const int nvec = (nq + 7) >> 3;
  const size_t v0 = (d.offset + (size_t)q0) >> 3;
  if (!mu_live(p, gb)) {   // the bucket is consumed here: zero it also on a skipped step
    if (p.raw)
      for (int k = threadIdx.x; k < nvec; k += kMuThreads) InVec<GDT>::zero(const_cast<void*>(p.grad), v0 + k);
    return;
  }
  const float inv_scale = p.raw ? (float)(1.0 / (double)p.scaler->scale) : 1.f;
  const float coef = clip_coef(p.clip_kind, p.clip_max_norm, p.scaler);
  bf16* X = p.x0 + d.x_offset;
  float sq = 0.f;
  for (int k = threadIdx.x; k < nvec; k += kMuThreads) {
    const size_t vi = v0 + k;
    const int valid = min(8, nq - 8 * k);   // the matrix's last vector may end in padding: left untouched
    float g[8], b[8];
    InVec<GDT>::load(p.grad, vi, g);
    if (p.acc != nullptr) {
      float a[8];
      InVec<STK_F32>::load(p.acc, vi, a);
#pragma unroll
      for (int e = 0; e < 8; ++e) g[e] += a[e];
    }
    InVec<STK_F32>::load(p.buf, vi, b);
    bf16 x[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      if (e >= valid) continue;
      const float gg = form_grad(g[e], p.raw != 0, p.grad_mul, inv_scale, p.clip_kind, coef, p.clip_value);
      b[e] = lerp_torch(b[e], gg, h.one_m_mom);                   // buf.lerp_(g, 1 - momentum)
      const float u = h.nesterov ? lerp_torch(gg, b[e], h.mom) : b[e];   // g.lerp(buf, momentum) | buf
      x[e] = __float2bfloat16_rn(u);                              // u.bfloat16()
      const float xf = __bfloat162float(x[e]);
      sq = fmaf(xf, xf, sq);
    }
    st_stream_f8(p.buf + vi * 8, b);
    const int64_t q = q0 + 8 * k;
    if (!d.transposed && valid == 8) {
      *reinterpret_cast<uint4*>(X + q) = *reinterpret_cast<const uint4*>(x);
    } else {
      for (int e = 0; e < valid; ++e) X[mu_xi(d, q + e)] = x[e];
    }
    if (p.raw) InVec<GDT>::zero(const_cast<void*>(p.grad), vi);
  }
  sq = block_reduce<false>(sq, s_red);
  if (threadIdx.x == 0) p.part[tile] = sq;
}

// ---- 2: per-matrix fold: the norm, the step count -------------------------------------------------------------------------
__global__ void __launch_bounds__(kMuThreads) k_mu_fold(const MuParams p) {
  const int j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (j >= p.n_params) return;   // whole warp
  const stk_muon_param_t& d = p.prm[j];
  const unsigned gb = p.pgroup[d.param];
  const bool live = mu_live(p, gb);
  const int ntile = (int)(((int64_t)d.rows * d.cols + kMuTile - 1) / kMuTile);
  float s = 0.f;
  if (live)
    for (int k = lane; k < ntile; k += 32) s += p.part[d.tile0 + k];
  s = warp_reduce<false>(s);
  if (lane != 0) return;
  MuScal o{1.f, 0};
  if (live) {
    // X.norm() of a bf16 tensor is rounded to bf16; .clamp(min=eps) keeps a NaN norm
    const float n = __bfloat162float(__float2bfloat16_rn(__fsqrt_rn(s)));
    const float eps = p.g[gb & 0x7f].eps;
    o.n = n < eps ? eps : n;
    o.flags = 1;
    p.steps[d.param] += 1;
  }
  p.scal[j] = o;
}

// ---- 3: X = bf16(X / n) ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kMuThreads) k_mu_scale(const MuParams p) {
  const int tile = blockIdx.x;
  const int j = mu_find<0>(p, tile);
  const stk_muon_param_t d = p.prm[j];
  const MuScal sc = p.scal[j];
  if (!(sc.flags & 1)) return;
  const int64_t q0 = (int64_t)(tile - d.tile0) * kMuTile;
  const int nq = (int)min((int64_t)kMuTile, (int64_t)d.rows * d.cols - q0);
  bf16* X = p.x0 + d.x_offset + q0;
  for (int k = threadIdx.x; 8 * k < nq; k += kMuThreads) {
    if (8 * k + 8 <= nq) {
      uint4 u = *reinterpret_cast<const uint4*>(X + 8 * k);
      bf16* x = reinterpret_cast<bf16*>(&u);
#pragma unroll
      for (int e = 0; e < 8; ++e) x[e] = __float2bfloat16_rn(__fdiv_rn(__bfloat162float(x[e]), sc.n));
      *reinterpret_cast<uint4*>(X + 8 * k) = u;
    } else {
      for (int e = 8 * k; e < nq; ++e) X[e] = __float2bfloat16_rn(__fdiv_rn(__bfloat162float(X[e]), sc.n));
    }
  }
}

// ---- 4: the Newton-Schulz GEMMs ----------------------------------------------------------------------------------------
// One kMm x kMk tile of a row-major operand (rows [r0, r0 + kMm) of a matrix with `rows` rows and `ld` = k extent
// columns, columns [k0, k0 + kMk)) into s[row][k]; out-of-range elements are zero.
__device__ __forceinline__ void mu_load_rows(bf16 (*s)[kLds], const bf16* src, int rows, int ld, int r0, int k0) {
  for (int v = threadIdx.x; v < kMm * kMk / 8; v += kMmThreads) {
    const int row = v >> 2, kv = (v & 3) * 8;
    const int gr = r0 + row, gk = k0 + kv;
    const bf16* q = src + (size_t)gr * ld + gk;
    uint4 u = make_uint4(0, 0, 0, 0);
    if (gr < rows) {
      if (gk + 8 <= ld && (reinterpret_cast<uintptr_t>(q) & 15) == 0) {
        u = *reinterpret_cast<const uint4*>(q);
      } else {
        bf16* x = reinterpret_cast<bf16*>(&u);
        for (int e = 0; e < 8 && gk + e < ld; ++e) x[e] = q[e];
      }
    }
    *reinterpret_cast<uint4*>(&s[row][kv]) = u;
  }
}

// The kMk x kMm tile (k rows [k0, k0 + kMk), columns [n0, n0 + kMm)) of a row-major rows x ld matrix, transposed into
// s[n][k]; out-of-range elements are zero.
__device__ __forceinline__ void mu_load_cols(bf16 (*s)[kLds], const bf16* src, int rows, int ld, int n0, int k0) {
  for (int v = threadIdx.x; v < kMm * kMk / 8; v += kMmThreads) {
    const int kr = v >> 3, nv = (v & 7) * 8;
    const int gk = k0 + kr, gn = n0 + nv;
    const bf16* q = src + (size_t)gk * ld + gn;
    uint4 u = make_uint4(0, 0, 0, 0);
    bf16* x = reinterpret_cast<bf16*>(&u);
    if (gk < rows) {
      if (gn + 8 <= ld && (reinterpret_cast<uintptr_t>(q) & 15) == 0) u = *reinterpret_cast<const uint4*>(q);
      else
        for (int e = 0; e < 8 && gn + e < ld; ++e) x[e] = q[e];
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) s[nv + e][kr] = x[e];
  }
}

__device__ __forceinline__ void mma_bf16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ uint32_t ld_pair(const bf16* s) { return *reinterpret_cast<const uint32_t*>(s); }

// MODE 0: A = X X^T; 1: B = b A + c A A; 2: X' = a X + B X.  `iter`: the Newton-Schulz step (X in x0 when even).
template <int MODE>
__global__ void __launch_bounds__(kMmThreads) k_mu_gemm(const MuParams p, int iter) {
  __shared__ __align__(16) bf16 sa[kMm][kLds];
  __shared__ __align__(16) bf16 sb[kMm][kLds];
  const int t = blockIdx.x;
  const int j = MODE == 2 ? mu_find<2>(p, t) : mu_find<1>(p, t);
  const stk_muon_param_t d = p.prm[j];
  if (!(p.scal[j].flags & 1)) return;
  const MuGroup& h = p.g[p.pgroup[d.param] & 0x7f];
  if (iter >= h.ns_steps) return;
  const int r = d.rows, c = d.cols;
  int tm, tn;
  if constexpr (MODE == 2) {
    const int ntn = (c + kMm - 1) / kMm, lt = t - d.full0;
    tm = lt / ntn;
    tn = lt % ntn;
  } else {
    const int lt = t - d.tri0;
    tm = (int)((sqrtf(8.f * lt + 1.f) - 1.f) * 0.5f);
    while (tm * (tm + 1) / 2 > lt) --tm;
    while ((tm + 1) * (tm + 2) / 2 <= lt) ++tm;
    tn = lt - tm * (tm + 1) / 2;
  }
  const bf16* xc = (iter & 1 ? p.x1 : p.x0) + d.x_offset;
  bf16* xn = (iter & 1 ? p.x0 : p.x1) + d.x_offset;
  const bf16* am = p.a + d.a_offset;
  bf16* bm = p.b + d.a_offset;
  const int K = MODE == 0 ? c : r;
  const int m0 = tm * kMm, n0 = tn * kMm;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wm = (warp >> 1) * 32, wn = (warp & 1) * 32;
  const int gq = lane >> 2, tq = (lane & 3) * 2;
  float acc[2][4][4];
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[mi][ni][e] = 0.f;

  for (int k0 = 0; k0 < K; k0 += kMk) {
    if constexpr (MODE == 0) {
      mu_load_rows(sa, xc, r, c, m0, k0);
      mu_load_rows(sb, xc, r, c, n0, k0);
    } else if constexpr (MODE == 1) {
      mu_load_rows(sa, am, r, r, m0, k0);
      mu_load_rows(sb, am, r, r, n0, k0);   // A is symmetric: column j of A is row j
    } else {
      mu_load_rows(sa, bm, r, r, m0, k0);
      mu_load_cols(sb, xc, r, c, n0, k0);
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < kMk; kk += 16) {
      uint32_t af[2][4];
#pragma unroll
      for (int mi = 0; mi < 2; ++mi) {
        const int rb = wm + mi * 16 + gq;
        af[mi][0] = ld_pair(&sa[rb][kk + tq]);
        af[mi][1] = ld_pair(&sa[rb + 8][kk + tq]);
        af[mi][2] = ld_pair(&sa[rb][kk + tq + 8]);
        af[mi][3] = ld_pair(&sa[rb + 8][kk + tq + 8]);
      }
#pragma unroll
      for (int ni = 0; ni < 4; ++ni) {
        const int cb = wn + ni * 8 + gq;
        const uint32_t b0 = ld_pair(&sb[cb][kk + tq]), b1 = ld_pair(&sb[cb][kk + tq + 8]);
#pragma unroll
        for (int mi = 0; mi < 2; ++mi) mma_bf16(acc[mi][ni], af[mi], b0, b1);
      }
    }
    __syncthreads();
  }

  const int ncols = MODE == 2 ? c : r;
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int i = m0 + wm + mi * 16 + gq + (e >> 1) * 8;
        const int jj = n0 + wn + ni * 8 + tq + (e & 1);
        if (i >= r || jj >= ncols) continue;
        const float v = acc[mi][ni][e];
        if constexpr (MODE == 2) {
          const size_t o = (size_t)i * c + jj;
          xn[o] = __float2bfloat16_rn(fmaf(h.a, __bfloat162float(xc[o]), v));   // addmm(X, B, X, beta=a)
        } else {
          if (tm == tn && i < jj) continue;   // the diagonal tile's upper half is the mirror of its lower half
          bf16 o;
          if constexpr (MODE == 0) o = __float2bfloat16_rn(v);
          else o = __float2bfloat16_rn(fmaf(h.c, v, h.b * __bfloat162float(am[(size_t)i * r + jj])));   // addmm(A, A, A, beta=b, alpha=c)
          bf16* out = MODE == 0 ? const_cast<bf16*>(am) : bm;
          out[(size_t)i * r + jj] = o;
          out[(size_t)jj * r + i] = o;
        }
      }
}

// ---- 5: the update, the low-precision copy ----------------------------------------------------------------------------------
__global__ void __launch_bounds__(kMuThreads) k_mu_apply(const MuParams p) {
  const int tile = blockIdx.x;
  const int j = mu_find<0>(p, tile);
  const stk_muon_param_t d = p.prm[j];
  if (!(p.scal[j].flags & 1)) return;
  const MuGroup& h = p.g[p.pgroup[d.param] & 0x7f];
  const bf16* X = (h.ns_steps & 1 ? p.x1 : p.x0) + d.x_offset;
  const float alpha = (float)(-(h.lr * d.lr_ratio));   // add_(X, alpha=-adjusted_lr)
  const int64_t q0 = (int64_t)(tile - d.tile0) * kMuTile;
  const int nq = (int)min((int64_t)kMuTile, (int64_t)d.rows * d.cols - q0);
  const int nvec = (nq + 7) >> 3;
  const size_t v0 = (d.offset + (size_t)q0) >> 3;
  for (int k = threadIdx.x; k < nvec; k += kMuThreads) {
    const size_t vi = v0 + k;
    const int valid = min(8, nq - 8 * k);
    float w[8];
    InVec<STK_F32>::load(p.master, vi, w);
    const int64_t q = q0 + 8 * k;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      if (e >= valid) continue;
      const float x = __bfloat162float(X[mu_xi(d, q + e)]);
      w[e] = fmaf(alpha, x, __fmul_rn(w[e], h.keep));   // mul_(1 - lr wd), then add_
    }
    st_stream_f8(p.master + vi * 8, w);
    if (p.lp != nullptr) {
      if (p.lp_dtype == STK_BF16) store_out<STK_BF16>(p.lp, vi, w);
      else store_out<STK_F32>(p.lp, vi, w);
    }
  }
}

template <int GDT>
void mu_launch(const MuParams& p, int n_tiles, int n_tri, int n_full, cudaStream_t s) {
  const unsigned warps_grid = (unsigned)((32ll * p.n_params + kMuThreads - 1) / kMuThreads);
  k_mu_prep<GDT><<<n_tiles, kMuThreads, 0, s>>>(p);
  k_mu_fold<<<warps_grid, kMuThreads, 0, s>>>(p);
  k_mu_scale<<<n_tiles, kMuThreads, 0, s>>>(p);
  for (int it = 0; it < p.max_ns; ++it) {
    k_mu_gemm<0><<<n_tri, kMmThreads, 0, s>>>(p, it);
    k_mu_gemm<1><<<n_tri, kMmThreads, 0, s>>>(p, it);
    k_mu_gemm<2><<<n_full, kMmThreads, 0, s>>>(p, it);
  }
  k_mu_apply<<<n_tiles, kMuThreads, 0, s>>>(p);
}

}  // namespace stk

using namespace stk;

extern "C" {

int stk_muon_step(stk_ctx* c, const stk_muon_args_t* a, void* stream) {
  STK_REQUIRE(c, c && a && a->hyper && a->params && a->param_group && a->steps && a->master && a->momentum_buffer &&
                     a->x0 && a->x1 && a->a && a->b && a->workspace && a->grad,
              "stk_muon_step: NULL argument");
  STK_REQUIRE(c, a->n_groups >= 1 && a->n_groups <= STK_MAX_GROUPS, "stk_muon_step: n_groups must be in [1, 8]");
  STK_REQUIRE(c, a->n_params >= 1 && a->n_tiles >= 1 && a->n_tri >= 1 && a->n_full >= 1, "stk_muon_step: no matrices");
  STK_REQUIRE(c, (reinterpret_cast<uintptr_t>(a->workspace) & 15) == 0, "stk_muon_step: workspace must be 16-byte aligned");
  STK_REQUIRE(c, ((reinterpret_cast<uintptr_t>(a->x0) | reinterpret_cast<uintptr_t>(a->x1) |
                   reinterpret_cast<uintptr_t>(a->a) | reinterpret_cast<uintptr_t>(a->b)) & 15) == 0,
              "stk_muon_step: X, A and B must be 16-byte aligned");
  STK_REQUIRE(c, a->grad_raw ? (a->grad_dtype == STK_BF16 || a->grad_dtype == STK_F32) : a->grad_dtype == STK_F32,
              "stk_muon_step: gradients must be a bf16 / fp32 raw bucket or fp32 main gradients");
  STK_REQUIRE(c, a->lp == nullptr || a->lp_dtype == STK_BF16 || a->lp_dtype == STK_F32, "stk_muon_step: lp dtype");
  STK_REQUIRE(c, a->clip_kind >= STK_CLIP_NONE && a->clip_kind <= STK_CLIP_VALUE, "stk_muon_step: clip kind");
  for (int gi = 0; gi < a->n_groups; ++gi)
    STK_REQUIRE(c, a->hyper[gi].ns_steps >= 0 && a->hyper[gi].ns_steps < 100, "stk_muon_step: ns_steps must be in [0, 100)");
  std::lock_guard<std::mutex> lk(c->mu);
  DeviceGuard g(c->device);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);

  MuParams p{};
  p.prm = a->params;
  p.n_params = a->n_params;
  p.pgroup = a->param_group;
  p.steps = a->steps;
  p.master = a->master;
  p.buf = a->momentum_buffer;
  p.x0 = static_cast<bf16*>(a->x0);
  p.x1 = static_cast<bf16*>(a->x1);
  p.a = static_cast<bf16*>(a->a);
  p.b = static_cast<bf16*>(a->b);
  p.scal = reinterpret_cast<MuScal*>(a->workspace);
  p.part = reinterpret_cast<float*>(static_cast<char*>(a->workspace) + size_t(a->n_params) * 16);
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
  p.max_ns = 0;
  for (int gi = 0; gi < a->n_groups; ++gi) {
    const stk_muon_hyper_t& h = a->hyper[gi];
    MuGroup& o = p.g[gi];
    o.lr = h.lr;
    o.one_m_mom = (float)(1.0 - h.momentum);
    o.mom = (float)h.momentum;
    o.keep = (float)(1.0 - h.lr * h.weight_decay);
    o.a = (float)h.ns_a;
    o.b = (float)h.ns_b;
    o.c = (float)h.ns_c;
    o.eps = __bfloat162float(__float2bfloat16_rn((float)h.eps));   // clamp(min=eps) on a bf16 tensor
    o.nesterov = h.nesterov;
    o.ns_steps = h.ns_steps;
    p.max_ns = h.ns_steps > p.max_ns ? h.ns_steps : p.max_ns;
  }
  const bool bf16g = a->grad_raw && a->grad_dtype == STK_BF16;
  ProfScope prof(c, 1, s);
  if (bf16g) mu_launch<STK_BF16>(p, a->n_tiles, a->n_tri, a->n_full, s);
  else mu_launch<STK_F32>(p, a->n_tiles, a->n_tri, a->n_full, s);
  STK_CUDA(c, cudaGetLastError());
  return STK_OK;
}

}  // extern "C"
