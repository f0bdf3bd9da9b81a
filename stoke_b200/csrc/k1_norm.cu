// k1_norm.cu -- the norm / inf pass when there is no cross-rank reduce to fuse it into (world == 1), and the in-place clip of
// reduced gradients for the stock-optimizer route.
//
//   k_grad_norm  : reads the raw gradient bucket ONCE (2 B/element for bf16), accumulates sum g^2 | max |g| | sum |g|^p and the
//                  inf/nan flag of x = (g [+ acc]) * mul / scale, one partial per block.  Writes nothing else: the fused
//                  optimizer step (k_optim_step, raw route) reads the bucket a second time -- from L2 when the bucket fits
//                  (loads here carry an L2 evict_last policy; H100's L2 is 50 MB) -- and zeroes it.  Replaces the W == 1
//                  form of k_grad_reduce on the training path: 2 + 30 B/element through HBM instead of 8 + 30 (no fp32
//                  main-grad round trip).
//   k_grad_norm_finish : one block behind k_grad_norm or the W == 1 k_grad_reduce: folds their block partials and
//                  finishes them into the state (grad_norm, found_inf).
//   k_grad_scale : grad *= clip coefficient, or clamp (clip_grad_norm_'s scaling pass / clip_grad_value_,
//                  torch/nn/utils/clip_grad.py) for optimizers the fused step does not cover.
#include <cstdlib>

#include "k1_common.cuh"

namespace stk {

__device__ __forceinline__ uint64_t policy_evict_last() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ uint4 ld16_keep(const void* p, uint64_t pol) {  // bypass L1, keep in L2
  uint4 v;
  asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p), "l"(pol));
  return v;
}

struct NormParams {
  const void* grad;
  const float* acc;
  size_t nvec;       // 8-element vectors
  float mul, norm_p;
  int norm_kind;
  uint32_t flags;
  int keep_l2;       // 1 (default; STK_NORM_L2_KEEP=0 disables): loads carry an L2 evict_last policy -- the fused step's second
                     // read of the bucket then partly hits L2: on H100 (50 MB L2) at ResNet-50 size (51 MB bf16 bucket) K2 is
                     // 7 us faster and this pass 2 us slower than without the hint (bench.py, H100 80GB HBM3 at 400 W)
  stk_scaler_state_t* scaler;
  float* blk_partial;
};

template <int IN_DT>
struct RawVec;  // the raw words of one 8-element vector (kept packed until use: 4 registers per 16-bit vector in flight)
template <>
struct RawVec<STK_F32> {
  uint4 a, b;
  __device__ void load(const void* base, size_t v, uint64_t pol, bool keep) {
    const uint4* q = reinterpret_cast<const uint4*>(base) + 2 * v;
    a = keep ? ld16_keep(q, pol) : ld_stream16(q);
    b = keep ? ld16_keep(q + 1, pol) : ld_stream16(q + 1);
  }
  __device__ void unpack(float (&f)[8]) const {
    f[0] = __uint_as_float(a.x); f[1] = __uint_as_float(a.y); f[2] = __uint_as_float(a.z); f[3] = __uint_as_float(a.w);
    f[4] = __uint_as_float(b.x); f[5] = __uint_as_float(b.y); f[6] = __uint_as_float(b.z); f[7] = __uint_as_float(b.w);
  }
};
template <int DT16>
struct RawVec16 {
  uint4 u;
  __device__ void load(const void* base, size_t v, uint64_t pol, bool keep) {
    const uint4* q = reinterpret_cast<const uint4*>(base) + v;
    u = keep ? ld16_keep(q, pol) : ld_stream16(q);
  }
  __device__ void unpack(float (&f)[8]) const { unpack16<DT16>(u, f); }
};
template <>
struct RawVec<STK_BF16> : RawVec16<STK_BF16> {};
template <>
struct RawVec<STK_F16> : RawVec16<STK_F16> {};

constexpr int kNormThreads = 256;
constexpr int kNormUnroll = 8;  // 8 independent 16-byte loads per thread: 32 KB in flight per block

// One-shot blocks (one tile of kNormThreads * kNormUnroll vectors each, the shape that streams best on this part,
// tools/membench.cu): load, reduce, write ONE partial, retire -- no ticket, no fence, no block waits on an atomic.  The
// partials are folded by k_grad_norm_finish, a single block launched right behind on the same stream (stream order is the
// only synchronisation), in a fixed order -> run-to-run deterministic.  k_grad_reduce at world 1 ends the same way.
template <int IN_DT, bool HAS_ACC>
__global__ void __launch_bounds__(kNormThreads) k_grad_norm(const NormParams p) {
  const uint64_t pol = policy_evict_last();
  float inv_scale = 1.f;
  if (p.flags & STK_RF_UNSCALE) inv_scale = (float)(1.0 / (double)p.scaler->scale);
  const float mul = p.mul;
  float part = 0.f;
  bool bad = false;
  const size_t t0 = size_t(blockIdx.x) * kNormThreads * kNormUnroll;
  RawVec<IN_DT> raw[kNormUnroll];
#pragma unroll
  for (int u = 0; u < kNormUnroll; ++u) {
    const size_t v = t0 + size_t(u) * kNormThreads + threadIdx.x;
    if (v < p.nvec) raw[u].load(p.grad, v, pol, p.keep_l2 != 0);
  }
#pragma unroll
  for (int u = 0; u < kNormUnroll; ++u) {
    const size_t v = t0 + size_t(u) * kNormThreads + threadIdx.x;
    if (v < p.nvec) {
      float g[8];
      raw[u].unpack(g);
      if (HAS_ACC) {
        float a[8];
        InVec<STK_F32>::load(p.acc, v, a);
#pragma unroll
        for (int i = 0; i < 8; ++i) g[i] += a[i];
      }
      fold8(g, mul, inv_scale, p.norm_kind, p.norm_p, part, bad);
    }
  }
  store_block_partial(p.blk_partial, p.norm_kind, part, bad);
}

// Folds the partials of k_grad_norm or of the world-1 k_grad_reduce (sign bit: the block saw inf/nan) in a fixed order and
// applies the bucket to the step accumulators.
__global__ void __launch_bounds__(1024) k_grad_norm_finish(const FinishParams f, unsigned nblocks) {
  __shared__ float s_red[32];
  const bool mx = f.norm_kind == STK_NORM_INF;
  float x = 0.f;
  bool bad = false;
  for (unsigned b = threadIdx.x; b < nblocks; b += blockDim.x) {
    float y = __ldcg(&f.blk_partial[b]);
    if (__float_as_uint(y) & 0x80000000u) {
      bad = true;
      y = fabsf(y);
    }
    x = mx ? fmax_nan(x, y) : x + y;
  }
  const float tot = mx ? block_reduce<true>(x, s_red) : block_reduce<false>(x, s_red);
  const int any_bad = __syncthreads_or(bad ? 1 : 0);
  if (threadIdx.x == 0) finish_bucket(f, tot, any_bad != 0);
}

cudaError_t launch_norm_finish(const FinishParams& f, unsigned nblocks, cudaStream_t s) {
  k_grad_norm_finish<<<1, 1024, 0, s>>>(f, nblocks);
  return cudaGetLastError();
}

__global__ void __launch_bounds__(256) k_grad_scale(float* __restrict__ grad, size_t nvec, int clip_kind, float max_norm,
                                                     float clip_value, const stk_scaler_state_t* scaler) {
  const size_t v = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (v >= nvec) return;
  float coef = 1.f;
  // a NaN norm gives a NaN coefficient and NaN gradients, as torch.clamp does in clip_grad_norm_
  if (clip_kind == STK_CLIP_NORM) coef = clamp_max_nan(max_norm / (scaler->grad_norm + 1e-6f), 1.0f);
  f8 g = ld_stream_f8(grad + v * 8);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    if (clip_kind == STK_CLIP_NORM) g.v[i] *= coef;
    else g.v[i] = clamp_nan(g.v[i], -clip_value, clip_value);
  }
  st_stream_f8(grad + v * 8, g.v);
}

}  // namespace stk

using namespace stk;

extern "C" {

int stk_grad_norm(stk_ctx* c, const void* grad, int grad_dtype, const float* acc, size_t n, double mul, int norm_kind,
                  double norm_p, unsigned flags, void* stream) {
  STK_REQUIRE(c, c && grad, "stk_grad_norm: NULL argument");
  STK_REQUIRE(c, n % 8 == 0, "stk_grad_norm: n must be a multiple of 8");
  STK_REQUIRE(c, norm_kind >= STK_NORM_NONE && norm_kind <= STK_NORM_P, "stk_grad_norm: bad norm kind");
  std::lock_guard<std::mutex> lk(c->mu);
  DeviceGuard g(c->device);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  NormParams p{};
  p.grad = grad;
  p.acc = acc;
  p.nvec = n / 8;
  p.mul = (float)mul;
  p.norm_p = (float)norm_p;
  p.norm_kind = norm_kind;
  p.flags = flags;
  {
    static int keep = -1;
    if (keep < 0) {
      const char* e = std::getenv("STK_NORM_L2_KEEP");
      keep = e ? std::atoi(e) : 1;
    }
    p.keep_l2 = keep;
  }
  p.scaler = c->scaler_dev;
  const size_t tile = size_t(kNormThreads) * kNormUnroll;
  size_t want = (p.nvec + tile - 1) / tile;
  if (want < 1) want = 1;
  void (*kern)(NormParams) = nullptr;
#define STK_PICK(DT) kern = acc ? k_grad_norm<DT, true> : k_grad_norm<DT, false>;
  switch (grad_dtype) {
    case STK_F32: STK_PICK(STK_F32) break;
    case STK_BF16: STK_PICK(STK_BF16) break;
    case STK_F16: STK_PICK(STK_F16) break;
    default: return stk_fail(c, STK_ERR_INVALID, "stk_grad_norm: bad dtype");
  }
#undef STK_PICK
  const unsigned grid = (unsigned)want;
  int rc = stk_grow_partials(c, grid, s);
  if (rc != STK_OK) return rc;
  p.blk_partial = c->blk_partial_dev;
  ProfScope prof(c, 3, s);
  kern<<<grid, kNormThreads, 0, s>>>(p);
  STK_CUDA(c, launch_norm_finish({p.blk_partial, c->accum_dev, p.scaler, p.norm_p, p.norm_kind, p.flags}, grid, s));
  return STK_OK;
}

int stk_grad_scale(stk_ctx* c, float* grad, size_t n, int clip_kind, double clip_max_norm, double clip_value, void* stream) {
  STK_REQUIRE(c, c && grad, "stk_grad_scale: NULL argument");
  STK_REQUIRE(c, n % 8 == 0, "stk_grad_scale: n must be a multiple of 8");
  STK_REQUIRE(c, clip_kind == STK_CLIP_NORM || clip_kind == STK_CLIP_VALUE, "stk_grad_scale: clip kind must be norm or value");
  if (n == 0) return STK_OK;
  DeviceGuard g(c->device);
  const size_t nvec = n / 8;
  k_grad_scale<<<(unsigned)((nvec + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      grad, nvec, clip_kind, (float)clip_max_norm, (float)clip_value, c->scaler_dev);
  STK_CUDA(c, cudaGetLastError());
  return STK_OK;
}

}  // extern "C"
