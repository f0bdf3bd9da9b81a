// k1_common.cuh -- pieces shared by the K1 kernels (k1_reduce.cu: register-staged loads, world 1 and cross-rank;
// k1_bulk.cu: bulk-async copies staged through shared memory; k1_nvls.cu: multimem; k1_norm.cu: the norm pass): launch
// parameters, typed 8-element vector access, the element fold (scale, inf/nan test, unscale, norm partial), the block
// partial the world-1 kernels hand to k_grad_norm_finish, the cross-rank tail (block partial -> end barrier carrying the
// partials -> in-kernel bucket zeroing -> ticket) and the norm / inf finalisation both of them end in.
#pragma once
#include "ctx.cuh"

namespace stk {

struct ReduceParams {
  PtrTable grad;      // W peer pointers to the gradient bucket
  PtrTable acc;       // W peer pointers to the fp32 local accumulators (p[0] == nullptr: none)
  PtrTable out;       // W peer pointers to the main-grad bucket
  const void* grad_mc;  // multicast mapping of the gradient bucket (multimem flavour only)
  void* out_mc;         // multicast mapping of the output bucket (multimem flavour, all-reduce mode)
  PeerPads pads;
  stk_scaler_state_t* scaler;
  StepAccum* accum;
  float* blk_partial;   // [grid] per-block norm partials (world 1)
  unsigned long long* prof_ns;  // optional {barrier-to-barrier ns, launches, zeroing-tail ns} (block 0), nullptr when off
  size_t vec_begin, vec_end;  // owned shard in units of 8 elements
  size_t vec_total, vec_per_shard;  // whole bucket / shard stride (for zeroing the local bucket after the end barrier)
  float mul;
  float norm_p;
  int rank, world, n_dst;
  int norm_kind;
  uint32_t flags;
  uint32_t epoch, aux_epoch;
};

// What k_grad_norm_finish needs to fold the block partials of a world-1 pass into the step.
struct FinishParams {
  const float* blk_partial;
  StepAccum* accum;
  stk_scaler_state_t* scaler;
  float norm_p;
  int norm_kind;
  uint32_t flags;
};

template <int DT>
struct InVec;  // 8 input elements -> 8 floats
template <>
struct InVec<STK_F32> {
  static constexpr int kBytes = 32;
  __device__ static void load(const void* base, size_t v, float (&f)[8]) {
    f8 a = ld_stream_f8(reinterpret_cast<const float*>(base) + v * 8);
#pragma unroll
    for (int i = 0; i < 8; ++i) f[i] = a.v[i];
  }
  __device__ static void zero(void* base, size_t v) {
    const float z[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    st_stream_f8(reinterpret_cast<float*>(base) + v * 8, z);
  }
};
template <int DT16>
struct InVec16 {
  static constexpr int kBytes = 16;
  __device__ static void load(const void* base, size_t v, float (&f)[8]) {
    unpack16<DT16>(ld_stream16(reinterpret_cast<const uint4*>(base) + v), f);
  }
  __device__ static void zero(void* base, size_t v) {
    st_stream16(reinterpret_cast<uint4*>(base) + v, make_uint4(0, 0, 0, 0));
  }
};
template <>
struct InVec<STK_BF16> : InVec16<STK_BF16> {};
template <>
struct InVec<STK_F16> : InVec16<STK_F16> {};

template <int DT>
__device__ __forceinline__ void store_out(void* base, size_t v, const float (&f)[8]) {
  if constexpr (DT == STK_F32) {
    st_stream_f8(reinterpret_cast<float*>(base) + v * 8, f);  // one 32-byte store: full sectors over NVLink
  } else {
    st_stream16(reinterpret_cast<uint4*>(base) + v,
                make_uint4(pack_bf16(f[0], f[1]), pack_bf16(f[2], f[3]), pack_bf16(f[4], f[5]), pack_bf16(f[6], f[7])));
  }
}

// The element step of every K1 kernel, for one 8-element vector of summed gradients: x = x * mul, inf/nan test,
// x *= inv_scale, then this thread's norm partial (sum x^2 | max |x| | sum |x|^p) of the fp32 value.  x returns the
// values the reduce kernels store.
__device__ __forceinline__ void fold8(float (&x)[8], float mul, float inv_scale, int norm_kind, float norm_p, float& part,
                                      bool& bad) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    float y = x[i] * mul;
    bad |= !finitef(y);
    y *= inv_scale;
    x[i] = y;
    if (norm_kind == STK_NORM_L2) part = fmaf(y, y, part);
    else if (norm_kind == STK_NORM_INF) part = fmax_nan(part, fabsf(y));
    else if (norm_kind == STK_NORM_P) part += __powf(fabsf(y), norm_p);
  }
}

// The optimizer's gradient from one stored element, shared by K2 (k2_optim.cu) and the LAMB / LARS steps
// (k2_layerwise.cu): a raw-bucket element (its accumulator already added) times mul and 1/loss_scale, then
// clip_grad_norm_'s coefficient (torch/nn/utils/clip_grad.py: max_norm / (total_norm + 1e-6), clamped to 1) or
// clip_grad_value_'s clamp.  Both clamps keep NaN like torch.clamp: a NaN norm (a NaN gradient without a loss scaler)
// makes every gradient NaN, as clip_grad_norm_ does, and clip by value passes a NaN element through.
__device__ __forceinline__ float clip_coef(int clip_kind, float clip_max_norm, const stk_scaler_state_t* scaler) {
  return clip_kind == STK_CLIP_NORM ? clamp_max_nan(clip_max_norm / (scaler->grad_norm + 1e-6f), 1.0f) : 1.f;
}
// g: the stored element; raw: it comes from a raw bucket (mul and inv_scale apply); coef: clip_coef's value
__device__ __forceinline__ float form_grad(float g, bool raw, float mul, float inv_scale, int clip_kind, float coef,
                                           float clip_value) {
  if (raw) {
    g *= mul;
    g *= inv_scale;
  }
  if (clip_kind == STK_CLIP_NORM) g *= coef;
  else if (clip_kind == STK_CLIP_VALUE) g = clamp_nan(g, -clip_value, clip_value);
  return g;
}

// torch.lerp(a, b, w) on fp32 (ATen/native/Lerp.h) with the FMA contraction nvcc gives torch's CUDA lerp kernels (the
// Tensor.lerp_ and foreach forms round alike): |w| < 0.5: a + w (b - a) -> FFMA(w, b - a, a);
// else b - (b - a)(1 - w) -> FFMA(-(b - a), 1 - w, b).  Shared by stk_weight_avg and the schedule-free step of K2.
__device__ __forceinline__ float lerp_torch(float a, float b, float w) {
  const float d = b - a;
  return fabsf(w) < 0.5f ? fmaf(w, d, a) : fmaf(-d, 1.f - w, b);
}

// World 1: the block's norm partial (fixed tree: run-to-run deterministic) into blk_partial[blockIdx.x], for
// k_grad_norm_finish launched behind the kernel on the same stream.  The sign bit carries the block's inf/nan verdict
// (partials are +0, positive, +inf or NaN for every norm kind); setting the bit keeps the magnitude, so an inf or NaN
// partial reaches the finisher as it is.  Must be called by all threads of the block.
__device__ __forceinline__ void store_block_partial(float* blk_partial, int norm_kind, float part, bool bad) {
  __shared__ float s_red[32];
  const float blk = norm_kind == STK_NORM_INF ? block_reduce<true>(part, s_red) : block_reduce<false>(part, s_red);
  const int any_bad = __syncthreads_or(bad ? 1 : 0);
  if (threadIdx.x == 0) blk_partial[blockIdx.x] = any_bad ? __uint_as_float(__float_as_uint(blk) | 0x80000000u) : blk;
}

// Folds one bucket's total (norm partial `tot`, inf/nan flag `inf`) into the step accumulators.  On STK_RF_FINAL it turns
// the running total into grad_norm and found_inf and resets the accumulators.  One thread.
__device__ __forceinline__ void finish_bucket(const FinishParams& f, float tot, bool inf) {
  float run = f.accum->norm_partial;  // running over the buckets of this optimizer step
  run = f.norm_kind == STK_NORM_INF ? fmax_nan(run, tot) : run + tot;
  uint32_t run_inf = f.accum->found_inf | (inf ? 1u : 0u);
  if (f.flags & STK_RF_FINAL) {
    // an inf / nan gradient gives what torch's clip_grad_norm_ returns: NaN if any element is NaN, else inf
    float norm = run;
    if (f.norm_kind == STK_NORM_L2) norm = sqrtf(run);
    else if (f.norm_kind == STK_NORM_P) norm = powf(run, 1.f / f.norm_p);
    f.scaler->grad_norm = norm;
    // the inf gate belongs to the loss scaler (GradScaler.step); without one the reference steps regardless
    f.scaler->found_inf = (run_inf && (f.flags & STK_RF_UNSCALE)) ? 1 : 0;
    run = 0.f;
    run_inf = 0;
  }
  f.accum->norm_partial = run;
  f.accum->found_inf = run_inf;
}

__host__ __device__ inline FinishParams finish_params(const ReduceParams& p) {
  return {p.blk_partial, p.accum, p.scaler, p.norm_p, p.norm_kind, p.flags};
}

// Everything after a cross-rank block's data phase.  `part` / `bad`: this thread's norm partial and inf/nan flag; t_begin:
// device timestamp taken after the start barrier (block 0 / thread 0, profiling only).  Must be called by all threads of
// the block.
template <int IN_DT, int W_T>
__device__ __forceinline__ void cross_rank_tail(const ReduceParams& p, float part, bool bad, unsigned long long t_begin) {
  static_assert(W_T != 1, "world 1 ends in store_block_partial + k_grad_norm_finish");
  __shared__ float s_red[32];
  __shared__ unsigned s_bad[32];
  const int W = W_T ? W_T : p.world;
  const bool mx = p.norm_kind == STK_NORM_INF;
  // ---- per-block partials (fixed tree: run-to-run deterministic); ONE block-wide barrier, then only warp 0 continues ----
  {
    const float wsum = mx ? warp_reduce<true>(part) : warp_reduce<false>(part);
    const unsigned wbad = __any_sync(0xffffffffu, bad);
    if ((threadIdx.x & 31) == 0) {
      s_red[threadIdx.x >> 5] = wsum;
      s_bad[threadIdx.x >> 5] = wbad;
    }
  }
  __syncthreads();

  // block partial (warp 0): needed before the end barrier, where it rides to the peers with the barrier flag
  float blk = 0.f;
  unsigned any_bad = 0;
  if (threadIdx.x < 32) {
    const unsigned nwarp = (blockDim.x + 31) >> 5;
    blk = threadIdx.x < nwarp ? s_red[threadIdx.x] : 0.f;
    blk = mx ? warp_reduce<true>(blk) : warp_reduce<false>(blk);
    any_bad = __any_sync(0xffffffffu, threadIdx.x < nwarp && s_bad[threadIdx.x] != 0);
  }

  // Publish this block's (norm partial, inf flag) to every rank BEFORE signalling the end barrier: the same thread then
  // does fence.sys + st.release of the flag, so whoever sees the flag sees the partial.  Every rank later sums all
  // W x grid partials in the same (rank, block) order -> bit-identical totals everywhere, with no third cross-GPU
  // round trip after the data phase.
  if (threadIdx.x < (unsigned)W) {
    RankScalars* slot = &p.pads.p[threadIdx.x]->blk_scal[p.rank][blockIdx.x];
    st_relaxed_sys_f32(&slot->norm_partial, blk);
    st_relaxed_sys_u32(&slot->found_inf, any_bad);
  }
  // a peer that never arrives: give up (error word is set, the host raises STK_ERR_PEER at its next call); nothing is
  // zeroed or finalised on top of an incomplete exchange
  if (!block_barrier_all_ranks(p.pads, p.rank, W, 1, p.epoch)) return;
  // end of the NVLink data phase (all peer reads and peer writes of this block are complete on every rank)
  unsigned long long t_data_end = 0;
  if (p.prof_ns && blockIdx.x == 0 && threadIdx.x == 0) t_data_end = globaltimer_ns();
  if (p.flags & STK_RF_ZERO_INPUT) {
    // Zero the LOCAL gradient bucket inside the kernel (no separate memset between backward and step).  Block b may only
    // clear what the peers' blocks b have finished reading -- exactly this block's own index pattern, replicated in every
    // shard: shard q of my bucket is read by rank q's block b at the same offsets, and that block has passed the end barrier.
    for (int q = 0; q < W; ++q) {
      const size_t qb = p.vec_per_shard * q;
      size_t qe = qb + p.vec_per_shard;
      if (qe > p.vec_total) qe = p.vec_total;
      for (size_t v = qb + size_t(blockIdx.x) * blockDim.x + threadIdx.x; v < qe; v += size_t(gridDim.x) * blockDim.x)
        InVec<IN_DT>::zero(p.grad.p[p.rank], v);
    }
  }
  if (p.prof_ns && blockIdx.x == 0 && threadIdx.x == 0) {
    atomicAdd(&p.prof_ns[0], t_data_end - t_begin);         // barrier-to-barrier: the NVLink phase
    atomicAdd(&p.prof_ns[1], 1ull);
    atomicAdd(&p.prof_ns[2], globaltimer_ns() - t_data_end);  // local (HBM) bucket-zeroing tail of block 0
  }

  // Only warp 0 stays for the bookkeeping: the other warps retire now, so a block never sits idle on the ticket's
  // fence + atomic round trip.
  if (threadIdx.x >= 32) return;
  const unsigned lane = threadIdx.x;
  // ---- plain ticket over the (<= SM count) co-resident blocks ----
  unsigned last = 0;
  if (lane == 0) {
    __threadfence();
    last = (atomicAdd(&p.accum->blocks_done, 1u) == gridDim.x - 1);
  }
  last = __shfl_sync(0xffffffffu, last, 0);
  if (!last) return;
  __threadfence();
  // every local block has passed its end barrier, so every peer block's partial has landed in this rank's pad
  float total = 0.f;
  unsigned inf = 0;
  for (int r = 0; r < W; ++r) {
    float x = 0.f;
    for (unsigned b = lane; b < gridDim.x; b += 32) {
      const RankScalars* slot = &p.pads.p[p.rank]->blk_scal[r][b];
      const float y = ld_relaxed_sys_f32(&slot->norm_partial);
      x = mx ? fmax_nan(x, y) : x + y;
      inf |= ld_relaxed_sys_u32(&slot->found_inf);
    }
    x = mx ? warp_reduce<true>(x) : warp_reduce<false>(x);
    total = mx ? fmax_nan(total, x) : total + x;
  }
  inf = __any_sync(0xffffffffu, inf != 0);
  if (lane == 0) {
    p.accum->blocks_done = 0;
    finish_bucket(finish_params(p), total, inf != 0);  // global values: every rank finishes the same totals
  }
}

// k1_norm.cu: folds `nblocks` partials written by store_block_partial into the step (one block, behind the kernel on `s`)
cudaError_t launch_norm_finish(const FinishParams& f, unsigned nblocks, cudaStream_t s);
// k1_bulk.cu: shared-memory / bulk-async flavour for cross-rank 16-bit buckets; cudaErrorNotSupported -> use k_grad_reduce
cudaError_t launch_reduce_bulk(stk_ctx* c, const ReduceParams& p, int grad_dtype, int out_dtype, int grid, cudaStream_t s);
// k1_nvls.cu: multimem (NVSwitch in-network reduction) flavour; cudaErrorNotSupported -> next flavour
cudaError_t launch_reduce_nvls(stk_ctx* c, const ReduceParams& p, int grad_dtype, int out_dtype, int grid, cudaStream_t s);

inline void coop_attr(stk_ctx* c, cudaLaunchConfig_t& cfg, cudaLaunchAttribute* attr) {
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = 1;
  cfg.attrs = attr;
  cfg.numAttrs = c->coop_launch ? 1 : 0;
}

}  // namespace stk
