// k2_optim.cu -- K2: single-pass fused optimizer step (Adam / AdamW / SGD-momentum / NAdam / RAdam / Adamax / Adadelta /
// Rprop / ASGD / Lion / schedule-free AdamW and SGD / AdEMAMix / TensorFlow-style RMSprop / Adan), plus the step prologues
// (per-parameter step counts, NAdam's mu_product, ASGD's eta and mu; the schedule-free group scalars; AdEMAMix's bias
// corrections and warm-ups; Adan's step sizes and first-step flags) and epilogue.
//
// One sweep over (grad, master, exp_avg, exp_avg_sq) does what the reference spreads over clip_grad_norm_'s scaling pass /
// clip_grad_value_, GradScaler.step's inf gate, the ~7 foreach kernels of torch.optim.Adam and (mixed precision) the
// fp32 -> bf16 parameter cast; in sharded (OSS / ZeRO-1) mode the updated low-precision shard is stored straight into
// every rank's parameter buffer, which is the parameter all-gather (K3).  HBM bytes per element: read g,p,m,v (16) +
// write p,m,v (12) [+ 2 for the bf16 copy] = 28 / 30, for every kind but SGD and ASGD (NAdam, RAdam, Adamax, Adadelta and
// Rprop keep two fp32 state tensors like Adam; Adamax's exp_inf, Adadelta's acc_delta and Rprop's step_size live in the
// exp_avg_sq buffer).  ASGD keeps one (ax, in exp_avg): read g,p,ax + write p,ax = 20 / 22, and 16 / 18 while mu == 1,
// when ax is written without being read.  Lion keeps one (exp_avg) and reads it: 20 / 22.  Schedule-free AdamW keeps
// z (exp_avg) and exp_avg_sq like Adam: 28 / 30; schedule-free SGD keeps z only: 20 / 22.  AdEMAMix keeps a third
// tensor (exp_avg_slow, in m2) besides exp_avg_fast and exp_avg_sq: 36 / 38, and 28 / 30 in a group with beta1 == 0,
// which neither reads nor writes exp_avg_fast.  RMSpropTF keeps square_avg (v), momentum_buffer (m) in a group with
// momentum and grad_avg (m2) in a centered group: 20 / 22 with neither, 28 / 30 with momentum, 36 / 38 with both.  Adan
// keeps four (exp_avg, exp_avg_sq, exp_avg_diff in m2 and neg_pre_grad in m3): 44 / 46.  The clip coefficient, the skip decision and the bias corrections come from device memory, so there is no host synchronisation anywhere on the
// step.
//
// Gradient sources:  MAIN  -- fp32 reduced / unscaled gradients written by K1 (cross-rank routes), indexed like the state;
//                    RAW   -- the local model-dtype bucket itself (+ optional fp32 accumulator), scaled by mul and 1/scale
//                             here and zeroed after the read: the world == 1 route (k_grad_norm supplies norm / inf), which
//                             drops the 6 B/element fp32 main-grad round trip.
// Layout extras: segments (the local state is the concatenation of this rank's shard of every gradient bucket) and a range
// table over the flat index space selecting the parameter group (per-group lr / betas / eps / weight decay ...) or skipping
// parameters that received no gradient this step (torch skips `p.grad is None`, torch/optim/optimizer.py).
//
// Arithmetic follows torch/optim/adam.py (_single_tensor_adam, the path torch takes on CPU -- the oracle),
// torch/optim/sgd.py (_single_tensor_sgd), nadam.py (_single_tensor_nadam), radam.py (_single_tensor_radam), adamax.py
// (_single_tensor_adamax), adadelta.py (_single_tensor_adadelta), rprop.py (_single_tensor_rprop) and asgd.py
// (_single_tensor_asgd); Lion follows stoke_b200.optim.Lion.step (torch has no Lion), the schedule-free kinds
// stoke_b200.optim.AdamWScheduleFree.step / SGDScheduleFree.step, AdEMAMix stoke_b200.optim.AdEMAMix.step,
// RMSpropTF stoke_b200.optim.RMSpropTF.step and Adan stoke_b200.optim.Adan.step, each rounded like those steps on CUDA; the clip follows
// torch/nn/utils/clip_grad.py:165-174 (coef = max_norm / (total_norm + 1e-6), clamped to 1) and :291-292 (clamp).
#include <cstdlib>

#include "ademamix.cuh"
#include "k1_common.cuh"

namespace stk {

struct GroupHyperD {   // host-side doubles, converted exactly like torch converts python scalars
  double lr, beta1, beta2, eps, weight_decay, momentum, dampening;
  int nesterov, maximize;
  double momentum_decay;  // NAdam
  int decoupled;          // NAdam / RAdam: decoupled weight decay; RMSpropTF: decoupled_decay; Adan: no_prox
  int centered;           // RMSpropTF (in the padding before rho, so that no field moves)
  double rho;                                    // Adadelta; RMSpropTF: alpha (the square_avg decay, like rho); Adan: beta3
  // Rprop's four; RMSpropTF keeps its momentum constants in the first two (stk_rmsprop_tf_step fills them)
  union {
    double etaminus;
    double buf_c;                                // RMSpropTF: momentum_buffer's addcdiv value (lr, or 1)
  };
  union {
    double etaplus;
    double upd_c;                                // RMSpropTF: the update's coefficient on momentum_buffer (1, or lr)
  };
  double step_size_min, step_size_max;
  double lambd, alpha, t0;                       // ASGD
};
struct GroupHyperS {   // what the inner loop reads (shared memory, one entry per parameter group)
  float b2, eps, wd, one_m_b1, one_m_b2, lr, one_m_damp, decay_mul, mom;
  int nesterov, maximize;
  float c0, c1, c2;  // the per-step scalars of step_scalars (the layout documented at stk_optim_step_prologue)
  int decoupled;
  // Adadelta's rho and Lion's beta1 share a slot: a wider struct changes every kind's shared-memory loads (and registers)
  union {
    float rho;                                  // Adadelta
    float b1;                                   // Lion
    int no_m1;                                  // AdEMAMix: beta1 == 0, exp_avg_fast is the gradient (no state)
    int centered;                               // RMSpropTF: the group keeps grad_avg
  };
  union {
    float one_m_rho;                            // Adadelta
    float c3;                                   // the fourth per-step scalar: schedule-free AdamW's fp32(1 / bc2),
                                                // AdEMAMix's 1 - beta3_t, Adan's first-step flag
    float one_m_alpha;                          // RMSpropTF: fp32(1 - alpha)
  };
  // Rprop's four; RMSpropTF keeps its momentum constants in the first three, Adan its beta3 in the first two
  union {
    float etaminus;
    float buf_c;                                // RMSpropTF: momentum_buffer's addcdiv value (lr, or 1)
    float b3;                                   // Adan: fp32(beta3)
  };
  union {
    float etaplus;
    float upd_c;                                // RMSpropTF: the update's coefficient on momentum_buffer (1, or lr)
    float one_m_b3;                             // Adan: fp32(1 - beta3)
  };
  union {
    float ss_min;
    int has_mom;                                // RMSpropTF: momentum > 0, the group keeps momentum_buffer
  };
  float ss_max;
};

struct OptimParams {
  float* master;
  float* m;
  float* v;
  const void* grad;     // MAIN: float*, local indexing.  RAW: model-dtype bucket, global indexing
  const float* acc;     // RAW only
  size_t nvec;          // 8-float vector count of the local state
  PtrTable lp;          // low-precision / remote parameter destinations (bases; indexed globally)
  void* lp_mc;          // multicast mapping of the parameter buffer: publish with ONE multimem.st instead of W peer stores
  unsigned long long* prof_ns;  // optional {ns between the barriers, launches} (block 0), nullptr when off
  int lp_world;         // 0: none
  int lp_rank_skip;     // lp dtype == f32 and destination == master's own buffer: skip that rank (aliased)
  const stk_scaler_state_t* scaler;
  PeerPads pads;
  int rank, world;
  uint32_t epoch;
  int cross_rank;       // 1: start/end block barriers around the peer stores
  int kind, clip_kind;
  float clip_max_norm, clip_value;
  float grad_mul;       // RAW
  int unscale;          // RAW: multiply by 1/loss_scale
  int any_mom;          // SGD: some group has momentum != 0 (the buffer is written)
  int n_groups;
  GroupHyperD g[STK_MAX_GROUPS];
  int n_seg;                                 // >= 1
  uint32_t seg_local[STK_MAX_SEGMENTS + 1];  // vector units
  uint32_t seg_global[STK_MAX_SEGMENTS];     // vector units
  int n_ranges;                              // 0: group 0 everywhere
  const uint32_t* range_end;                 // device, ascending, vector units (global)
  const uint8_t* range_group;                // device; bit 7: skip
  const float4* range_bc;                    // device, optional: per-range scalars of stk_optim_step_prologue
  const float4* group_bc;                    // device, optional: per-group scalars of stk_optim_step_prologue
  // appended, so that the fields above keep their offsets (and the other kinds their code)
  float* m2;                                 // AdEMAMix: exp_avg_slow; RMSpropTF: grad_avg (nullptr: no centered group)
  int m_deferred;                            // AdEMAMix: some group has beta1 == 0, so m is loaded once the range is known;
                                             // RMSpropTF: likewise, some group has no momentum
  int m2_deferred;                           // RMSpropTF: some group is not centered, so m2 is loaded once the range is
                                             // known (in the tail padding: the struct keeps its size)
  float* m3;                                 // Adan: neg_pre_grad (the block grows from 1984 to 1992 bytes)
};

// floats of per-entry scalar state the prologue carries (the stk_optim_step_prologue `scalar_state` array)
__host__ __device__ constexpr int scalar_state_width(int kind) {
  return kind == STK_OPT_NADAM ? 1 : (kind == STK_OPT_ASGD ? 2 : 0);
}

// Per-step scalars of the update of step t (the float4 layout documented at stk_optim_step_prologue), in double from the
// python-scalar formulas of torch's single-tensor functions.  st: the entry's scalar state before the step on entry, after
// it on return (fp32, like torch's tensors): NAdam's mu_product; ASGD's {eta, mu}; not touched for the other kinds.
__device__ __forceinline__ float4 step_scalars(int kind, const GroupHyperD& h, double t, float* st) {
  // SGD: the first step seeds the momentum buffer; Rprop: step_size = full_like(p, lr) at the first step
  if (kind == STK_OPT_SGD || kind == STK_OPT_ADADELTA || kind == STK_OPT_RPROP)
    return make_float4(0.f, 0.f, t == 1.0 ? 1.f : 0.f, 0.f);
  if (kind == STK_OPT_ASGD) {  // torch/optim/asgd.py: the update uses the STORED eta and mu, then both advance
    float eta = st[0], mu = st[1];
    if (t == 1.0) {  // lazy state initialisation: eta = lr (fp32 tensor), mu = 1
      eta = (float)h.lr;
      mu = 1.f;
    }
    const float4 o = make_float4(-eta, (float)(1.0 - h.lambd * (double)eta), mu, 0.f);
    st[0] = (float)(h.lr / pow(1.0 + h.lambd * h.lr * t, h.alpha));  // lr / ((1 + lambd lr step) ** alpha)
    st[1] = (float)(t - h.t0 > 1.0 ? 1.0 / (t - h.t0) : 1.0);      // 1 / max(1, step - t0)
    return o;
  }
  const double bc1 = 1.0 - pow(h.beta1, t);
  const double bc2 = 1.0 - pow(h.beta2, t);
  if (kind == STK_OPT_ADAM || kind == STK_OPT_ADAMW)  // torch/optim/adam.py:531-547: step_size, bias_correction2_sqrt
    return make_float4((float)(h.lr / bc1), (float)sqrt(bc2), t == 1.0 ? 1.f : 0.f, 0.f);
  if (kind == STK_OPT_NADAM) {  // torch/optim/nadam.py: mu, mu_next, mu_product *= mu, the two addcdiv_ values
    const double mu = h.beta1 * (1.0 - 0.5 * pow(0.96, t * h.momentum_decay));
    const double mu_next = h.beta1 * (1.0 - 0.5 * pow(0.96, (t + 1.0) * h.momentum_decay));
    const float prod = __fmul_rn(*st, (float)mu);  // fp32 tensor times a python float
    *st = prod;
    const double prod_next = (double)prod * mu_next;
    return make_float4((float)(-h.lr * (1.0 - mu) / (1.0 - (double)prod)), (float)(-h.lr * mu_next / (1.0 - prod_next)),
                       (float)bc2, 0.f);
  }
  if (kind == STK_OPT_RADAM) {  // torch/optim/radam.py: rho_inf, rho_t, rect, the rectified and the plain update
    const double rho_inf = 2.0 / (1.0 - h.beta2) - 1.0;
    const double rho_t = rho_inf - 2.0 * t * pow(h.beta2, t) / bc2;
    if (rho_t > 5.0) {
      const double rect = sqrt((rho_t - 4.0) * (rho_t - 2.0) * rho_inf / ((rho_inf - 4.0) * (rho_inf - 2.0) * rho_t));
      return make_float4((float)(h.lr * rect * sqrt(bc2) / bc1), 1.f, 0.f, 0.f);
    }
    return make_float4((float)(h.lr / bc1), 0.f, 0.f, 0.f);
  }
  // none: only the step count advances (the schedule-free scalars come from k_sf_prologue)
  if (kind >= STK_OPT_LION) return make_float4(0.f, 0.f, 0.f, 0.f);
  return make_float4((float)(h.lr / bc1), 0.f, 0.f, 0.f);  // Adamax: clr = lr / bias_correction
}

// local vector index -> global vector index
__device__ __forceinline__ size_t to_global(const OptimParams& p, size_t i) {
  if (p.n_seg == 1) return p.seg_global[0] + (i - p.seg_local[0]);
  int lo = 0, hi = p.n_seg - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (p.seg_local[mid] <= i) lo = mid;
    else hi = mid - 1;
  }
  return p.seg_global[lo] + (i - p.seg_local[lo]);
}
// global vector index -> range index (first j with range_end[j] > gv)
__device__ __forceinline__ int range_of(const OptimParams& p, size_t gv) {
  int lo = 0, hi = p.n_ranges - 1;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(&p.range_end[mid]) > gv) hi = mid;
    else lo = mid + 1;
  }
  return lo;
}

template <int LP_DT, int VPT>  // -1: none, STK_BF16, STK_F32;  VPT vectors (8 elements each), adjacent in memory
__device__ __forceinline__ void store_lp(const OptimParams& p, size_t gv, const float (&x)[VPT][8], int nv) {
  if constexpr (LP_DT == STK_BF16) {
    uint4 u[VPT];
#pragma unroll
    for (int k = 0; k < VPT; ++k)
      u[k] = make_uint4(pack_bf16(x[k][0], x[k][1]), pack_bf16(x[k][2], x[k][3]), pack_bf16(x[k][4], x[k][5]),
                        pack_bf16(x[k][6], x[k][7]));
    if (p.lp_mc != nullptr) {
      // the NVSwitch replicates the store into every rank's parameter buffer (this rank's own copy included)
#pragma unroll
      for (int k = 0; k < VPT; ++k)
        if (k < nv) mm_st16(reinterpret_cast<uint4*>(p.lp_mc) + gv + k, u[k]);
      return;
    }
#pragma unroll 1
    for (int d = 0; d < p.lp_world; ++d) {
      const int dst = p.lp_world == 1 ? 0 : (p.rank + d) % p.lp_world;
      uint4* q = reinterpret_cast<uint4*>(p.lp.p[dst]) + gv;
      if (VPT == 2 && nv == 2) {
        // the thread's whole 32-byte sector, as two back-to-back 16-byte stores (sm_90's widest global store)
        st_stream16(q, u[0]);
        st_stream16(q + 1, u[VPT - 1]);
      } else {
        st_stream16(q, u[0]);
      }
    }
  } else if constexpr (LP_DT == STK_F32) {
#pragma unroll 1
    for (int d = 0; d < p.lp_world; ++d) {
      const int dst = p.lp_world == 1 ? 0 : (p.rank + d) % p.lp_world;
      if (dst == p.lp_rank_skip) continue;
#pragma unroll
      for (int k = 0; k < VPT; ++k)
        if (k < nv) st_stream_f8(reinterpret_cast<float*>(p.lp.p[dst]) + (gv + k) * 8, x[k]);
    }
  }
}

// GRAD: STK_F32 with RAW = false -> MAIN.  RAW = true -> the raw bucket of dtype GRAD.
// PERSIST = false: one-shot launch, VPT vectors per thread (local step; tools/membench.cu compares it with a persistent
// grid-stride loop).  PERSIST = true: co-resident grid-stride loop, required when the kernel
// pushes its shard to peers and therefore carries the cross-rank block barriers (sharded / OSS step).
// The kinds after SGD ask for two co-resident blocks per SM: left to themselves, ptxas caps ASGD's paired sharded form at
// 80 registers and NAdam's and RAdam's unpaired sharded forms at 64, and spills (ASGD's conditional ax load); with the
// bound none spills.  A minimum of 0 is no minimum: Adam, AdamW and SGD compile exactly as with __launch_bounds__(256).
template <int KIND, int LP_DT, bool PERSIST, int VPT, int GRAD, bool RAW>
__global__ void __launch_bounds__(256, KIND >= STK_OPT_NADAM ? 2 : 0) k_optim_step(const OptimParams p) {
  __shared__ GroupHyperS s_g[STK_MAX_GROUPS];
  __shared__ int s_skip;
  __shared__ float s_inv_scale;
  if (PERSIST && p.cross_rank && !block_barrier_all_ranks(p.pads, p.rank, p.world, 0, p.epoch)) return;
  unsigned long long t_begin = 0;
  if (PERSIST && p.prof_ns && blockIdx.x == 0 && threadIdx.x == 0) t_begin = globaltimer_ns();

  // SGD without momentum, AdEMAMix with beta1 == 0 and RMSpropTF without momentum in every group have no m
  const bool use_m = (KIND != STK_OPT_SGD && KIND != STK_OPT_ADEMAMIX && KIND != STK_OPT_RMSPROP_TF) || p.m != nullptr;
  // ASGD, Lion and schedule-free SGD: one state tensor (ax / exp_avg / z, in p.m)
  constexpr bool kHasV = KIND != STK_OPT_SGD && KIND != STK_OPT_ASGD && KIND != STK_OPT_LION && KIND != STK_OPT_SF_SGD;
  constexpr bool kHasM2 = KIND == STK_OPT_ADEMAMIX || KIND == STK_OPT_RMSPROP_TF || KIND == STK_OPT_ADAN;
  constexpr bool kHasM3 = KIND == STK_OPT_ADAN;
  constexpr bool kDeferM = KIND == STK_OPT_ADEMAMIX || KIND == STK_OPT_RMSPROP_TF;   // m may exist in some groups only
  const size_t stride = PERSIST ? size_t(gridDim.x) * blockDim.x * VPT : 0;
  size_t i = (size_t(blockIdx.x) * blockDim.x + threadIdx.x) * VPT;

  float g[VPT][8], w[VPT][8], m[VPT][8], v[VPT][8];
  float m2[kHasM2 ? VPT : 1][8];
  float m3[kHasM3 ? VPT : 1][8];
  size_t gv = 0;
  int nv = 0;
  auto load = [&]() {
    // issue this thread's loads before the (serial, double-precision) bias-correction prologue so that the pow()
    // latency hides behind the memory latency: 32 bytes per stream and vector (two 16-byte loads), all in flight together
    nv = (i + VPT <= p.nvec) ? VPT : (i < p.nvec ? 1 : 0);
    if (nv == 0) return;
    gv = to_global(p, i);
#pragma unroll
    for (int k = 0; k < VPT; ++k)
      if (k < nv) {
        if constexpr (RAW) InVec<GRAD>::load(p.grad, gv + k, g[k]);
        else InVec<STK_F32>::load(p.grad, i + k, g[k]);
        InVec<STK_F32>::load(p.master, i + k, w[k]);
        // ASGD: ax only when mu != 1; AdEMAMix with a beta1 == 0 group: m only where beta1 != 0; RMSpropTF likewise m
        // where the group has momentum and m2 where it is centered
        if (use_m && KIND != STK_OPT_ASGD && !(kDeferM && p.m_deferred)) InVec<STK_F32>::load(p.m, i + k, m[k]);
        if (kHasV) InVec<STK_F32>::load(p.v, i + k, v[k]);
        if constexpr (kHasM2) {
          if (KIND == STK_OPT_ADEMAMIX || KIND == STK_OPT_ADAN || (p.m2 != nullptr && !p.m2_deferred))
            InVec<STK_F32>::load(p.m2, i + k, m2[k]);
        }
        if constexpr (kHasM3) InVec<STK_F32>::load(p.m3, i + k, m3[k]);
      }
    if constexpr (RAW) {
      if (p.acc != nullptr) {
#pragma unroll
        for (int k = 0; k < VPT; ++k)
          if (k < nv) {
            float a[8];
            InVec<STK_F32>::load(p.acc, gv + k, a);
#pragma unroll
            for (int e = 0; e < 8; ++e) g[k][e] += a[e];
          }
      }
    }
  };
  load();

  if (threadIdx.x == 0) {
    s_skip = p.scaler->found_inf != 0;  // GradScaler.step: no optimizer.step() at all when any grad is inf/nan
    s_inv_scale = (RAW && p.unscale) ? (float)(1.0 / (double)p.scaler->scale) : 1.f;
  }
  if (threadIdx.x < (unsigned)p.n_groups) {
    const GroupHyperD& h = p.g[threadIdx.x];
    GroupHyperS o;
    // the per-step scalars: stk_optim_step_prologue's when given; else Adam / AdamW / SGD form the optimizer-wide step's
    // here (in double, ahead of the rest so that the pow() latency overlaps the loads) and the kinds after SGD take range_bc
    float4 c = make_float4(0.f, 0.f, 0.f, 0.f);
    if constexpr (KIND <= STK_OPT_SGD) c = step_scalars(KIND, h, (double)(p.scaler->opt_steps + 1), nullptr);
    if (p.group_bc != nullptr) c = p.group_bc[threadIdx.x];
    o.c0 = c.x;
    o.c1 = c.y;
    o.c2 = c.z;
    o.b2 = (float)h.beta2;
    o.eps = (float)h.eps;
    o.wd = (float)h.weight_decay;
    o.one_m_b1 = (float)(1.0 - h.beta1);
    o.one_m_b2 = (float)(1.0 - h.beta2);
    o.lr = (float)h.lr;
    o.one_m_damp = (float)(1.0 - h.dampening);
    o.decay_mul = (float)(1.0 - h.lr * h.weight_decay);  // AdamW: param.mul_(1 - lr * wd)
    o.mom = (float)h.momentum;
    o.nesterov = h.nesterov;
    o.maximize = h.maximize;
    o.decoupled = h.decoupled;
    if constexpr (KIND == STK_OPT_ADADELTA) {
      o.rho = (float)h.rho;
      o.one_m_rho = (float)(1.0 - h.rho);
    }
    if constexpr (KIND == STK_OPT_RPROP) {
      o.etaminus = (float)h.etaminus;
      o.etaplus = (float)h.etaplus;
      o.ss_min = (float)h.step_size_min;
      o.ss_max = (float)h.step_size_max;
    }
    if constexpr (KIND == STK_OPT_LION) o.b1 = (float)h.beta1;
    if constexpr (KIND == STK_OPT_SF_ADAMW || KIND == STK_OPT_SF_SGD || KIND == STK_OPT_ADEMAMIX || KIND == STK_OPT_ADAN)
      o.c3 = c.w;
    if constexpr (KIND == STK_OPT_ADEMAMIX) o.no_m1 = h.beta1 == 0.0;
    if constexpr (KIND == STK_OPT_RMSPROP_TF) {
      o.one_m_alpha = (float)(1.0 - h.rho);
      o.centered = h.centered;
      o.decay_mul = (float)__dadd_rn(1.0, -__dmul_rn(h.lr, h.weight_decay));   // python's 1 - lr * wd, not one DFMA
      o.has_mom = h.momentum > 0.0;
      o.buf_c = (float)h.buf_c;
      o.upd_c = (float)h.upd_c;
    }
    if constexpr (KIND == STK_OPT_ADAN) {
      o.b1 = (float)h.beta1;
      o.b3 = (float)h.rho;
      o.one_m_b3 = (float)(1.0 - h.rho);
      // python's 1 - lr * wd (no_prox, a multiplier) or 1 + lr * wd (a divisor: torch's CUDA division by a python
      // scalar b multiplies by fp32(1 / b), the reciprocal taken in double), without a DFMA
      const double lr_wd = __dmul_rn(h.lr, h.weight_decay);
      o.decay_mul = (float)(h.decoupled ? __dadd_rn(1.0, -lr_wd) : __ddiv_rn(1.0, __dadd_rn(1.0, lr_wd)));
    }
    s_g[threadIdx.x] = o;
  }
  __syncthreads();
  const bool skip_all = s_skip != 0;
  const float coef = clip_coef(p.clip_kind, p.clip_max_norm, p.scaler);
  const float cv = p.clip_value;
  const float inv_scale = s_inv_scale;

  while (nv > 0) {
    unsigned rb = 0;
    float4 bc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (p.n_ranges > 0) {  // the VPT vectors of a thread never straddle a parameter (16-element alignment)
      const int rj = range_of(p, gv);
      rb = __ldg(&p.range_group[rj]);
      if (p.range_bc != nullptr) bc = __ldg(&p.range_bc[rj]);
    }
    GroupHyperS h = s_g[rb & 0x7f];
    if (p.range_bc != nullptr) {  // per-parameter step counts (torch's `state[p]["step"]`)
      h.c0 = bc.x;
      h.c1 = bc.y;
      h.c2 = bc.z;
      if constexpr (KIND == STK_OPT_ADEMAMIX || KIND == STK_OPT_ADAN) h.c3 = bc.w;
    }
    const bool skip = skip_all || (rb & 0x80u);
    if (!skip) {
#pragma unroll
      for (int k = 0; k < VPT; ++k) {
        if (k >= nv) continue;
        if constexpr (KIND == STK_OPT_ASGD) {  // ax is only read when it is averaged (torch: mu.item() != 1)
          if (h.c2 != 1.f) InVec<STK_F32>::load(p.m, i + k, m[k]);
        }
        if constexpr (KIND == STK_OPT_ADEMAMIX) {  // exp_avg_fast does not exist in a beta1 == 0 group
          if (p.m_deferred && !h.no_m1) InVec<STK_F32>::load(p.m, i + k, m[k]);
        }
        if constexpr (KIND == STK_OPT_RMSPROP_TF) {  // momentum_buffer / grad_avg exist only with momentum / centered
          if (p.m_deferred && h.has_mom) InVec<STK_F32>::load(p.m, i + k, m[k]);
          if (p.m2_deferred && h.centered) InVec<STK_F32>::load(p.m2, i + k, m2[k]);
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          float gg = form_grad(g[k][e], RAW, p.grad_mul, inv_scale, p.clip_kind, coef, cv);
          if (h.maximize) gg = -gg;
          float ww = w[k][e];
          if (KIND == STK_OPT_ADAM || KIND == STK_OPT_ADAMW) {
            if (KIND == STK_OPT_ADAMW) ww *= h.decay_mul;
            else if (h.wd != 0.f) gg = fmaf(ww, h.wd, gg);          // grad.add(param, alpha=wd)
            float mm = m[k][e];
            mm = fmaf(h.one_m_b1, gg - mm, mm);                      // exp_avg.lerp_(grad, 1 - beta1)
            float vv = v[k][e] * h.b2;
            vv = fmaf(h.one_m_b2 * gg, gg, vv);                      // mul_(beta2).addcmul_(grad, grad, value=1-beta2)
            const float denom = sqrtf(vv) / h.c1 + h.eps;            // c1 = bias_correction2_sqrt
            ww = ww - h.c0 * (mm / denom);                           // addcdiv_(exp_avg, denom, value=-step_size)
            m[k][e] = mm;
            v[k][e] = vv;
          } else if (KIND == STK_OPT_NADAM || KIND == STK_OPT_RADAM) {
            if (h.wd != 0.f) {
              if (h.decoupled) ww *= h.decay_mul;                    // param.mul_(1 - lr * wd)
              else gg = fmaf(ww, h.wd, gg);                          // grad.add(param, alpha=wd)
            }
            float mm = m[k][e];
            mm = fmaf(h.one_m_b1, gg - mm, mm);                      // exp_avg.lerp_(grad, 1 - beta1)
            float vv = v[k][e] * h.b2;
            vv = fmaf(h.one_m_b2 * gg, gg, vv);                      // mul_(beta2).addcmul_(grad, grad, value=1-beta2)
            if (KIND == STK_OPT_NADAM) {
              const float denom = sqrtf(vv / h.c2) + h.eps;          // exp_avg_sq.div(bc2).sqrt().add_(eps)
              ww = fmaf(h.c0, gg / denom, ww);                       // addcdiv_(grad, denom, value=c_g)
              ww = fmaf(h.c1, mm / denom, ww);                       // addcdiv_(exp_avg, denom, value=c_m)
            } else if (h.c1 != 0.f) {                                // rho_t > 5: rectified adaptive step
              ww = ww - h.c0 * (mm / (sqrtf(vv) + h.eps));
            } else {                                                 // unrectified: SGD with momentum
              ww = ww - h.c0 * mm;
            }
            m[k][e] = mm;
            v[k][e] = vv;
          } else if (KIND == STK_OPT_ADAMAX) {
            if (h.wd != 0.f) gg = fmaf(ww, h.wd, gg);               // grad.add(param, alpha=wd)
            float mm = m[k][e];
            mm = fmaf(h.one_m_b1, gg - mm, mm);                      // exp_avg.lerp_(grad, 1 - beta1)
            // torch.maximum(exp_inf.mul_(beta2), grad.abs().add_(eps)): NaN-propagating, unlike fmaxf
            const float uu = fmax_nan(v[k][e] * h.b2, fabsf(gg) + h.eps);
            ww = ww - h.c0 * (mm / uu);                              // addcdiv_(exp_avg, exp_inf, value=-clr)
            m[k][e] = mm;
            v[k][e] = uu;
          } else if (KIND == STK_OPT_ADADELTA) {
            if (h.wd != 0.f) gg = fmaf(ww, h.wd, gg);               // grad.add(param, alpha=wd)
            const float sq = fmaf(h.one_m_rho * gg, gg, m[k][e] * h.rho);  // square_avg.mul_(rho).addcmul_(g, g, 1-rho)
            // delta = acc_delta.add(eps).sqrt_().div_(square_avg.add(eps).sqrt_()).mul_(grad)
            const float dl = sqrtf(v[k][e] + h.eps) / sqrtf(sq + h.eps) * gg;
            v[k][e] = fmaf(h.one_m_rho * dl, dl, v[k][e] * h.rho);  // acc_delta.mul_(rho).addcmul_(delta, delta, 1-rho)
            m[k][e] = sq;
            ww = fmaf(-h.lr, dl, ww);                                // param.add_(delta, alpha=-lr)
          } else if (KIND == STK_OPT_RPROP) {
            // first step: prev = zeros, step_size = full_like(p, lr) with the lr in force now; V is not used then
            const bool first = h.c2 != 0.f;
            const float prev = first ? 0.f : m[k][e];
            float ss = first ? h.lr : v[k][e];
            const float x = gg * prev;                               // grad.mul(prev).sign(): the fp32 product's sign
            float f = (float)((x > 0.f) - (x < 0.f));                // torch.sign: NaN and +-0 give 0
            if (f > 0.f) f = h.etaplus;                              // sign[sign.gt(0)] = etaplus
            if (f < 0.f) f = h.etaminus;                             // sign[sign.lt(0)] = etaminus
            if (f == 0.f) f = 1.f;                                   // sign[sign.eq(0)] = 1
            ss = ss * f;                                             // step_size.mul_(sign).clamp_(min, max), NaN kept
            ss = ss < h.ss_min ? h.ss_min : ss;
            ss = ss > h.ss_max ? h.ss_max : ss;
            if (f == h.etaminus) gg = 0.f;                           // grad[sign.eq(etaminus)] = 0
            const float sg = (float)((gg > 0.f) - (gg < 0.f));
            ww = ww - sg * ss;                                       // param.addcmul_(grad.sign(), step_size, value=-1)
            m[k][e] = gg;                                            // prev.copy_(grad)
            v[k][e] = ss;
          } else if (KIND == STK_OPT_ASGD) {
            if (h.wd != 0.f) gg = fmaf(ww, h.wd, gg);               // grad.add(param, alpha=wd)
            ww = fmaf(h.c0, gg, __fmul_rn(ww, h.c1));                // param.mul_(1 - lambd eta).add_(grad, alpha=-eta)
            // ax.add_(param.sub(ax).mul_(mu)), or ax.copy_(param) while mu == 1
            m[k][e] = h.c2 == 1.f ? ww : __fadd_rn(m[k][e], __fmul_rn(ww - m[k][e], h.c2));
          } else if (KIND == STK_OPT_LION) {
            if (h.wd != 0.f) ww *= h.decay_mul;                     // param.mul_(1 - lr * wd), before the update
            const float mm = m[k][e];
            // exp_avg.mul(beta1).add_(g, alpha=1 - beta1): torch's CUDA add(alpha) contracts to one FFMA
            const float c = fmaf(gg, h.one_m_b1, __fmul_rn(mm, h.b1));
            const float sg = (float)((c > 0.f) - (c < 0.f));       // .sign_(): NaN and +-0 give 0
            ww = fmaf(-h.lr, sg, ww);                                // param.add_(u, alpha=-lr)
            m[k][e] = fmaf(gg, h.one_m_b2, __fmul_rn(mm, h.b2));    // exp_avg.mul_(beta2).add_(g, alpha=1 - beta2)
          } else if (KIND == STK_OPT_SF_ADAMW || KIND == STK_OPT_SF_SGD) {
            // group scalars (k_sf_prologue): c0 = ckp1, c1 = lr (beta1 (1 - ckp1) - 1), c2 = lr, c3 = fp32(1 / bc2)
            float d = gg;
            if (KIND == STK_OPT_SF_ADAMW) {
              // exp_avg_sq.mul_(beta2).addcmul_(g, g, value=1 - beta2): torch's CUDA addcmul rounds g * g first
              const float vv = fmaf(h.one_m_b2, __fmul_rn(gg, gg), __fmul_rn(v[k][e], h.b2));
              // exp_avg_sq.mul(1 / bc2).sqrt_().add_(eps), then g / denom
              d = __fdiv_rn(gg, __fadd_rn(__fsqrt_rn(__fmul_rn(vv, h.c3)), h.eps));
              v[k][e] = vv;
            }
            if (h.wd != 0.f) d = fmaf(ww, h.wd, d);                 // d.add(y, alpha=wd), y before this step's update
            ww = lerp_torch(ww, m[k][e], h.c0);                      // y.lerp_(z, ckp1)
            ww = fmaf(h.c1, d, ww);                                  // y.add_(d, alpha=lr (beta1 (1 - ckp1) - 1))
            m[k][e] = fmaf(-h.c2, d, m[k][e]);                       // z.sub_(d, alpha=lr)
          } else if (KIND == STK_OPT_ADEMAMIX) {
            // per-step scalars (k_ademamix_prologue): c0 = 1 / bc1, c1 = 1 / sqrt(bc2), c2 = alpha_t, c3 = 1 - beta3_t
            const float mf = h.no_m1 ? gg : lerp_torch(m[k][e], gg, h.one_m_b1);  // exp_avg_fast.lerp_(g, 1 - beta1)
            const float ms = lerp_torch(m2[k][e], gg, h.c3);                     // exp_avg_slow.lerp_(g, 1 - beta3_t)
            // exp_avg_sq.mul_(beta2).addcmul_(g, g, value=1 - beta2): torch's CUDA addcmul rounds g * g first
            const float vv = fmaf(h.one_m_b2, __fmul_rn(gg, gg), __fmul_rn(v[k][e], h.b2));
            // exp_avg_sq.sqrt().mul_(1 / sqrt(bc2)).add_(eps)
            const float den = __fadd_rn(__fmul_rn(__fsqrt_rn(vv), h.c1), h.eps);
            // exp_avg_fast.mul(1 / bc1).add_(exp_avg_slow, alpha=alpha_t).div_(denom): add(alpha) is one FFMA
            float u = __fdiv_rn(fmaf(ms, h.c2, __fmul_rn(mf, h.c0)), den);
            if (h.wd != 0.f) u = fmaf(ww, h.wd, u);                   // u.add_(p, alpha=weight_decay)
            ww = fmaf(-h.lr, u, ww);                                 // p.add_(u, alpha=-lr)
            m[k][e] = mf;
            m2[k][e] = ms;
            v[k][e] = vv;
          } else if (KIND == STK_OPT_RMSPROP_TF) {
            if (h.wd != 0.f) {
              if (h.decoupled) ww = __fmul_rn(ww, h.decay_mul);      // p.mul_(1 - lr * wd)
              else gg = fmaf(h.wd, ww, gg);                          // grad = grad.add(p, alpha=wd)
            }
            // square_avg.add_(grad.pow(2) - square_avg, alpha=1 - alpha): pow(2) is g * g, add(alpha) one FFMA
            const float sq = fmaf(h.one_m_alpha, __fsub_rn(__fmul_rn(gg, gg), v[k][e]), v[k][e]);
            float avg;
            if (h.centered) {
              const float ga = fmaf(h.one_m_alpha, __fsub_rn(gg, m2[k][e]), m2[k][e]);  // grad_avg.add_(g - ga, 1 - alpha)
              // square_avg.addcmul(grad_avg, grad_avg, value=-1).add(eps).sqrt_(): addcmul rounds ga * ga first
              avg = __fsqrt_rn(__fadd_rn(__fsub_rn(sq, __fmul_rn(ga, ga)), h.eps));
              m2[k][e] = ga;
            } else {
              avg = __fsqrt_rn(__fadd_rn(sq, h.eps));                // square_avg.add(eps).sqrt_()
            }
            const float q = __fdiv_rn(gg, avg);
            if (h.has_mom) {
              // buf.mul_(momentum).addcdiv_(grad, avg, value=c): addcdiv is one FFMA on the quotient
              const float buf = fmaf(h.buf_c, q, __fmul_rn(m[k][e], h.mom));
              ww = fmaf(-h.upd_c, buf, ww);                          // p.add_(-buf) | p.add_(buf, alpha=-lr)
              m[k][e] = buf;
            } else {
              ww = fmaf(-h.lr, q, ww);                               // p.addcdiv_(grad, avg, value=-lr)
            }
            v[k][e] = sq;
          } else if (KIND == STK_OPT_ADAN) {
            // per-step scalars (k_adan_prologue): c0 = lr / bc1, c1 = lr beta2 / bc2, c2 = 1 / sqrt(bc3),
            // c3 = first (neg_pre_grad = -g, so the first difference is 0)
            const float x = __fadd_rn(h.c3 != 0.f ? -gg : m3[k][e], gg);       // P.add_(g): g - g_prev
            const float mm = fmaf(gg, h.one_m_b1, __fmul_rn(m[k][e], h.b1));   // exp_avg.mul_(b1).add_(g, alpha=1 - b1)
            const float dd = fmaf(x, h.one_m_b2, __fmul_rn(m2[k][e], h.b2));   // exp_avg_diff likewise with P, beta2
            const float u = __fadd_rn(__fmul_rn(x, h.b2), gg);                 // P.mul_(beta2).add_(g)
            // exp_avg_sq.mul_(beta3).addcmul_(P, P, value=1 - beta3): addcmul rounds P * P first
            const float nn = fmaf(h.one_m_b3, __fmul_rn(u, u), __fmul_rn(v[k][e], h.b3));
            const float den = __fadd_rn(__fmul_rn(__fsqrt_rn(nn), h.c2), h.eps);  // (sqrt(n) / sqrt(bc3)).add_(eps)
            if (h.decoupled) ww = __fmul_rn(ww, h.decay_mul);                   // no_prox: p.mul_(1 - lr wd)
            ww = fmaf(-h.c0, __fdiv_rn(mm, den), ww);                           // addcdiv is one FFMA on the quotient
            ww = fmaf(-h.c1, __fdiv_rn(dd, den), ww);
            if (!h.decoupled) ww = __fmul_rn(ww, h.decay_mul);                  // p.div_(1 + lr wd)
            m[k][e] = mm;
            m2[k][e] = dd;
            v[k][e] = nn;
            m3[k][e] = __fadd_rn(0.f, -gg);                                     // P.zero_().add_(g, alpha=-1)
          } else {  // SGD
            if (h.wd != 0.f) gg = fmaf(ww, h.wd, gg);
            if (h.mom != 0.f) {
              const float bb = h.c2 != 0.f ? gg : fmaf(m[k][e], h.mom, h.one_m_damp * gg);  // first step: buf = g
              m[k][e] = bb;
              gg = h.nesterov ? fmaf(bb, h.mom, gg) : bb;
            }
            ww = fmaf(-h.lr, gg, ww);
          }
          w[k][e] = ww;
        }
      }
#pragma unroll
      for (int k = 0; k < VPT; ++k)
        if (k < nv) {
          st_stream_f8(p.master + (i + k) * 8, w[k]);
          if (use_m && (KIND != STK_OPT_SGD || p.any_mom) && !(KIND == STK_OPT_ADEMAMIX && h.no_m1) &&
              !(KIND == STK_OPT_RMSPROP_TF && !h.has_mom))
            st_stream_f8(p.m + (i + k) * 8, m[k]);
          if (kHasV) st_stream_f8(p.v + (i + k) * 8, v[k]);
          if constexpr (kHasM2) {
            if (KIND == STK_OPT_ADEMAMIX || KIND == STK_OPT_ADAN || h.centered) st_stream_f8(p.m2 + (i + k) * 8, m2[k]);
          }
          if constexpr (kHasM3) st_stream_f8(p.m3 + (i + k) * 8, m3[k]);
        }
      store_lp<LP_DT, VPT>(p, gv, w, nv);
    }
    if constexpr (RAW) {
      // the bucket is consumed (also on a skipped step): zero it for the next backward's in-place accumulation
#pragma unroll
      for (int k = 0; k < VPT; ++k)
        if (k < nv) InVec<GRAD>::zero(const_cast<void*>(p.grad), gv + k);
    }
    if (!PERSIST) break;
    i += stride;
    load();
  }
  if (PERSIST && p.cross_rank) block_barrier_all_ranks(p.pads, p.rank, p.world, 1, p.epoch);
  if (PERSIST && p.prof_ns && blockIdx.x == 0 && threadIdx.x == 0) {
    atomicAdd(&p.prof_ns[0], globaltimer_ns() - t_begin);
    atomicAdd(&p.prof_ns[1], 1ull);
  }
}

struct StepPrologueParams {
  GroupHyperD g[STK_MAX_GROUPS];
  int n_groups, n_ranges, kind;
  const uint8_t* range_group;
  int32_t* range_steps;
  float* scalar_state;
  float4* bc;
  const stk_scaler_state_t* scaler;
};

// The step-count bookkeeping every prologue shares: one thread per range (n_ranges > 0) or per group (n_ranges == 0).
// The entry's group, the steps it has taken (its own count, or the optimizer-wide one), and whether this step advances it:
// not when the range is skipped or the step found inf (torch increments state[p]["step"] only for parameters that are
// stepped).  False when the thread has no entry.
struct StepEntry {
  int j;
  unsigned group;
  int64_t done;
  bool advance, per_range;
};
__device__ __forceinline__ bool step_entry(int n_groups, int n_ranges, const uint8_t* range_group,
                                           const int32_t* range_steps, const stk_scaler_state_t* scaler, StepEntry& e) {
  e.j = blockIdx.x * blockDim.x + threadIdx.x;
  e.per_range = n_ranges > 0;
  if (e.j >= (e.per_range ? n_ranges : n_groups)) return false;
  const unsigned b = e.per_range ? (unsigned)range_group[e.j] : (unsigned)e.j;
  e.group = b & 0x7f;
  e.done = e.per_range ? (int64_t)range_steps[e.j] : scaler->opt_steps;
  e.advance = !(b & 0x80u) && scaler->found_inf == 0;
  return true;
}
// after an advancing step: the entry's own count moves (the optimizer-wide one is the epilogue's)
__device__ __forceinline__ void step_entry_advance(const StepEntry& e, int32_t* range_steps) {
  if (e.per_range) range_steps[e.j] = (int32_t)(e.done + 1);
}

// the scalars of each entry's NEXT step and, when it advances, its step count and scalar state (NAdam's mu_product,
// ASGD's eta and mu)
__global__ void k_step_prologue(const StepPrologueParams p) {
  StepEntry e;
  if (!step_entry(p.n_groups, p.n_ranges, p.range_group, p.range_steps, p.scaler, e)) return;
  const int j = e.j;
  const int w = scalar_state_width(p.kind);
  float st[2] = {1.f, 1.f};
  for (int k = 0; k < w; ++k) st[k] = p.scalar_state[j * w + k];
  p.bc[j] = step_scalars(p.kind, p.g[e.group], (double)(e.done + 1), st);
  if (!e.advance) return;
  for (int k = 0; k < w; ++k) p.scalar_state[j * w + k] = st[k];
  step_entry_advance(e, p.range_steps);
}

struct AdemamixPrologueParams {
  double beta1[STK_MAX_GROUPS], beta2[STK_MAX_GROUPS];
  stk_ademamix_hyper_t a[STK_MAX_GROUPS];
  int n_groups, n_ranges;
  const uint8_t* range_group;
  int32_t* range_steps;
  float4* bc;
  const stk_scaler_state_t* scaler;
};

// stk_optim_step_prologue's bookkeeping with AdEMAMix's scalars (no scalar state)
__global__ void k_ademamix_prologue(const AdemamixPrologueParams p) {
  StepEntry e;
  if (!step_entry(p.n_groups, p.n_ranges, p.range_group, p.range_steps, p.scaler, e)) return;
  p.bc[e.j] = ademamix_scalars(p.beta1[e.group], p.beta2[e.group], p.a[e.group], (double)(e.done + 1));
  if (e.advance) step_entry_advance(e, p.range_steps);
}

struct AdanPrologueParams {
  double lr[STK_MAX_GROUPS], beta1[STK_MAX_GROUPS], beta2[STK_MAX_GROUPS];
  stk_adan_hyper_t a[STK_MAX_GROUPS];
  int n_groups, n_ranges;
  const uint8_t* range_group;
  int32_t* range_steps;
  float4* bc;
  const stk_scaler_state_t* scaler;
};

// stk_optim_step_prologue's bookkeeping with Adan.step's scalars.  The bias corrections use the optimizer-wide count (Adan
// keeps `step` in the group); an entry's own count only says whether it has a previous gradient.  In python doubles and
// python's order (the explicit roundings keep nvcc from contracting, which python does not do):
// {lr / bc1, lr * beta2 / bc2, 1 / sqrt(bc3), first}
__global__ void k_adan_prologue(const AdanPrologueParams p) {
  StepEntry e;
  if (!step_entry(p.n_groups, p.n_ranges, p.range_group, p.range_steps, p.scaler, e)) return;
  const unsigned gi = e.group;
  const int64_t done = p.scaler->opt_steps;
  const double t = (double)(done + 1);
  const double bc1 = __dadd_rn(1.0, -pow(p.beta1[gi], t));
  const double bc2 = __dadd_rn(1.0, -pow(p.beta2[gi], t));
  const double bc3 = __dadd_rn(1.0, -pow(p.a[gi].beta3, t));
  const bool first = done == 0 || e.done == 0;   // upstream: "neg_pre_grad" not in state or group["step"] == 1
  p.bc[e.j] = make_float4((float)__ddiv_rn(p.lr[gi], bc1), (float)__ddiv_rn(__dmul_rn(p.lr[gi], p.beta2[gi]), bc2),
                          (float)__ddiv_rn(1.0, __dsqrt_rn(bc3)), first ? 1.f : 0.f);
  if (e.advance) step_entry_advance(e, p.range_steps);
}

struct SfPrologueParams {
  stk_sf_hyper_t g[STK_MAX_GROUPS];
  int n_groups;
  double* state;   // {lr_max, weight_sum} per group
  float4* bc;
  const stk_scaler_state_t* scaler;
};

// One thread per group: the schedule-free group scalars of step k + 1 (AdamWScheduleFree.step / SGDScheduleFree.step, in
// python doubles; the explicit roundings keep nvcc from contracting a * b - 1 into one DFMA, which python does not do)
// and, unless found_inf, the advance of lr_max and weight_sum.  k itself is the optimizer-wide count, advanced by the
// epilogue only on a step that was applied.
__global__ void k_sf_prologue(const SfPrologueParams p) {
  const int j = threadIdx.x;
  if (j >= p.n_groups) return;
  const stk_sf_hyper_t& h = p.g[j];
  const int64_t k = p.scaler->opt_steps;
  const double kp1 = (double)(k + 1);
  const double sched = k < h.warmup_steps ? __ddiv_rn(kp1, (double)h.warmup_steps) : 1.0;
  const double lr = __dmul_rn(h.lr, sched);
  const double prev_max = p.state[2 * j];
  const double lr_max = prev_max > lr ? prev_max : lr;                     // python max(lr, lr_max)
  const double weight = __dmul_rn(pow(kp1, h.r), pow(lr_max, h.weight_lr_power));
  const double weight_sum = __dadd_rn(p.state[2 * j + 1], weight);
  const double ckp1 = weight_sum != 0.0 ? __ddiv_rn(weight, weight_sum) : 0.0;
  const double y_lr = __dmul_rn(lr, __dadd_rn(__dmul_rn(h.beta1, __dadd_rn(1.0, -ckp1)), -1.0));
  const double bc2 = __dadd_rn(1.0, -pow(h.beta2, kp1));
  p.bc[j] = make_float4((float)ckp1, (float)y_lr, (float)lr, (float)__ddiv_rn(1.0, bc2));
  if (p.scaler->found_inf != 0) return;
  p.state[2 * j] = lr_max;
  p.state[2 * j + 1] = weight_sum;
}

// scaler.update() (torch/amp/grad_scaler.py:549-556 -> _amp_update_scale_), step counters, per-step accumulator reset
__global__ void k_step_epilogue(stk_scaler_state_t* st, StepAccum* acc) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const bool inf = st->found_inf != 0;
  if (inf) st->skipped_steps += 1;
  else st->opt_steps += 1;
  if (st->enabled) {
    if (inf) {
      st->scale = st->scale * st->backoff_factor;
      st->growth_tracker = 0;
    } else {
      int t = st->growth_tracker + 1;
      if (t == st->growth_interval) {
        float ns = st->scale * st->growth_factor;
        if (finitef(ns)) st->scale = ns;   // _amp_update_scale_: do not grow past the largest finite fp32
        t = 0;
      }
      st->growth_tracker = t;
    }
  }
  st->found_inf = 0;
  acc->norm_partial = 0.f;
  acc->found_inf = 0u;
}

}  // namespace stk

using namespace stk;

static void fill_groups(GroupHyperD* o, const stk_optim_hyper_t* h, const stk_optim_hyper_ext_t* ext, int n) {
  for (int gi = 0; gi < n; ++gi) {
    o[gi].lr = h[gi].lr; o[gi].beta1 = h[gi].beta1; o[gi].beta2 = h[gi].beta2; o[gi].eps = h[gi].eps;
    o[gi].weight_decay = h[gi].weight_decay; o[gi].momentum = h[gi].momentum; o[gi].dampening = h[gi].dampening;
    o[gi].nesterov = h[gi].nesterov; o[gi].maximize = h[gi].maximize;
    o[gi].momentum_decay = ext ? ext[gi].momentum_decay : 0.0;
    o[gi].decoupled = ext ? (ext[gi].decoupled_weight_decay != 0) : 0;
    o[gi].rho = ext ? ext[gi].rho : 0.0;
    o[gi].etaminus = ext ? ext[gi].etaminus : 0.0;
    o[gi].etaplus = ext ? ext[gi].etaplus : 0.0;
    o[gi].step_size_min = ext ? ext[gi].step_size_min : 0.0;
    o[gi].step_size_max = ext ? ext[gi].step_size_max : 0.0;
    o[gi].lambd = ext ? ext[gi].lambd : 0.0;
    o[gi].alpha = ext ? ext[gi].alpha : 0.0;
    o[gi].t0 = ext ? ext[gi].t0 : 0.0;
  }
}

static size_t g_grid_nvec = 0;  // set under the context lock by stk_optim_step_ex (cross-rank launches only)

template <typename K>
static cudaError_t launch_one(stk_ctx* c, K kernel, const OptimParams& p, bool persist, int vpt, cudaStream_t s) {
  const size_t per_block = size_t(256) * vpt;
  const size_t nvec = (persist && g_grid_nvec) ? g_grid_nvec : p.nvec;  // same grid on every rank
  size_t grid = (nvec + per_block - 1) / per_block;  // one-shot: VPT vectors per thread
  if (grid < 1) grid = 1;
  if (persist) {  // co-resident grid-stride loop: at most two blocks per SM
    size_t res = (size_t)std::min(blocks_per_sm(c, kernel, 256), 2) * c->sm_count;
    if (res > (size_t)kMaxBlocks) res = kMaxBlocks;
    if (grid > res) grid = res;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3(256);
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  coop_attr(c, cfg, attr);
  if (!persist) cfg.numAttrs = 0;
  ProfScope prof(c, 1, s);
  return cudaLaunchKernelEx(&cfg, kernel, p);
}

template <int KIND>
static cudaError_t launch_optim(stk_ctx* c, const OptimParams& p, int lp_dtype, int grad_dtype, bool raw, bool pair,
                                cudaStream_t s) {
  if (raw) {
    // raw route: local step only (world == 1)
    if (grad_dtype == STK_BF16 && p.lp_world == 1 && lp_dtype == STK_BF16)
      return launch_one(c, k_optim_step<KIND, STK_BF16, false, 1, STK_BF16, true>, p, false, 1, s);
    if (grad_dtype == STK_F32 && p.lp_world == 0)
      return launch_one(c, k_optim_step<KIND, -1, false, 1, STK_F32, true>, p, false, 1, s);
    return cudaErrorNotSupported;
  }
  if (p.cross_rank) {
    if (lp_dtype == STK_BF16) {
      // Adan's four state streams spill in two vectors per thread under __launch_bounds__(256, 2): one vector only
      if constexpr (KIND != STK_OPT_ADAN) {
        if (pair && p.lp_mc == nullptr) return launch_one(c, k_optim_step<KIND, STK_BF16, true, 2, STK_F32, false>, p, true, 2, s);
      }
      return launch_one(c, k_optim_step<KIND, STK_BF16, true, 1, STK_F32, false>, p, true, 1, s);
    }
    return launch_one(c, k_optim_step<KIND, STK_F32, true, 1, STK_F32, false>, p, true, 1, s);
  }
  if (p.lp_world == 0) return launch_one(c, k_optim_step<KIND, -1, false, 1, STK_F32, false>, p, false, 1, s);
  if (lp_dtype == STK_BF16) return launch_one(c, k_optim_step<KIND, STK_BF16, false, 1, STK_F32, false>, p, false, 1, s);
  return launch_one(c, k_optim_step<KIND, STK_F32, false, 1, STK_F32, false>, p, false, 1, s);
}

// The body of stk_optim_step_ex, stk_rmsprop_tf_step and stk_adan_step: rt is the RMSPROP_TF groups' array, ad the ADAN
// groups' array and m3 ADAN's neg_pre_grad (nullptr for every other kind, which the callers check)
static int optim_step(stk_ctx* c, const stk_optim_args_t* a, const stk_rmsprop_tf_hyper_t* rt,
                      const stk_adan_hyper_t* ad, float* m3, void* stream) {
  STK_REQUIRE(c, c && a && a->hyper && a->master && a->grad, "stk_optim_step_ex: NULL argument");
  STK_REQUIRE(c, a->n_groups >= 1 && a->n_groups <= STK_MAX_GROUPS, "stk_optim_step_ex: n_groups must be in [1, 8]");
  STK_REQUIRE(c, a->n_local % 8 == 0, "stk_optim_step_ex: n_local must be a multiple of 8");
  const stk_optim_hyper_t* h = a->hyper;
  STK_REQUIRE(c, h->kind >= STK_OPT_ADAM && h->kind <= STK_OPT_ADAN, "stk_optim_step_ex: bad optimizer kind");
  const bool sf = h->kind == STK_OPT_SF_ADAMW || h->kind == STK_OPT_SF_SGD;
  const bool ademamix = h->kind == STK_OPT_ADEMAMIX;
  const bool rmsprop_tf = h->kind == STK_OPT_RMSPROP_TF;
  const bool adan = h->kind == STK_OPT_ADAN;
  STK_REQUIRE(c, !adan || a->group_bc || (a->n_ranges > 0 && a->range_bc),
              "stk_adan_step: needs the scalars of stk_adan_step_prologue (group_bc or range_bc)");
  STK_REQUIRE(c, !adan || (a->exp_avg && a->exp_avg_sq && a->exp_avg_slow && m3),
              "stk_adan_step: needs exp_avg, exp_avg_sq, exp_avg_slow (exp_avg_diff) and neg_pre_grad");
  STK_REQUIRE(c, !sf || a->group_bc, "stk_optim_step_ex: the schedule-free kinds need group_bc of stk_sf_step_prologue");
  STK_REQUIRE(c, h->kind <= STK_OPT_SGD || h->kind == STK_OPT_LION || rmsprop_tf || a->group_bc ||
                     (a->n_ranges > 0 && a->range_bc),
              "stk_optim_step_ex: the kinds after SGD need the scalars of stk_optim_step_prologue (group_bc or range_bc)");
  STK_REQUIRE(c, (reinterpret_cast<uintptr_t>(a->group_bc) & 15) == 0, "stk_optim_step_ex: group_bc must be 16-byte aligned");
  STK_REQUIRE(c, h->kind == STK_OPT_SGD || ademamix || rmsprop_tf ||
                     (a->exp_avg && (a->exp_avg_sq || h->kind == STK_OPT_ASGD || h->kind == STK_OPT_LION ||
                                     h->kind == STK_OPT_SF_SGD)),
              "stk_optim_step_ex: this kind needs exp_avg and exp_avg_sq (ASGD, Lion, SF_SGD: exp_avg)");
  bool any_mom = false, any_b1 = false, any_b1_zero = false, any_centered = false, any_plain = false;
  bool any_rms_mom = false, any_rms_no_mom = false;
  for (int gi = 0; gi < a->n_groups; ++gi) {
    STK_REQUIRE(c, h[gi].kind == h->kind, "stk_optim_step_ex: all groups must use the same optimizer kind");
    any_mom |= h[gi].momentum != 0.0;
    any_b1 |= h[gi].beta1 != 0.0;
    any_b1_zero |= h[gi].beta1 == 0.0;
    if (rmsprop_tf) {
      any_rms_mom |= h[gi].momentum > 0.0;
      any_rms_no_mom |= !(h[gi].momentum > 0.0);
      any_centered |= rt[gi].centered != 0;
      any_plain |= rt[gi].centered == 0;
    }
  }
  STK_REQUIRE(c, !ademamix || (a->exp_avg_slow && a->exp_avg_sq && (a->exp_avg || !any_b1)),
              "stk_optim_step_ex: ADEMAMIX needs exp_avg_slow, exp_avg_sq and (unless every group has beta1 == 0) exp_avg");
  STK_REQUIRE(c, !rmsprop_tf || (a->exp_avg_sq && (a->exp_avg || !any_rms_mom) && (a->exp_avg_slow || !any_centered)),
              "stk_rmsprop_tf_step: needs exp_avg_sq, exp_avg when some group has momentum > 0 and exp_avg_slow when "
              "some group is centered");
  STK_REQUIRE(c, !(h->kind == STK_OPT_SGD && any_mom && !a->exp_avg), "stk_optim_step_ex: SGD momentum needs a buffer");
  STK_REQUIRE(c, a->lp_ptrs == nullptr || a->lp_world == 1 || a->lp_world == c->world, "stk_optim_step_ex: lp_world must be 1 or world");
  STK_REQUIRE(c, a->lp_ptrs == nullptr || a->lp_dtype == STK_BF16 || a->lp_dtype == STK_F32, "stk_optim_step_ex: lp dtype");
  STK_REQUIRE(c, a->n_seg >= 0 && a->n_seg <= STK_MAX_SEGMENTS, "stk_optim_step_ex: too many segments");
  STK_REQUIRE(c, a->n_seg == 0 || (a->seg_local && a->seg_global), "stk_optim_step_ex: segment arrays are NULL");
  STK_REQUIRE(c, a->n_ranges == 0 || (a->range_end_vec && a->range_group), "stk_optim_step_ex: range arrays are NULL");
  STK_REQUIRE(c, !a->grad_raw || c->world == 1 || a->lp_world <= 1, "stk_optim_step_ex: the raw gradient route is local (no peer stores)");
  STK_REQUIRE(c, a->grad_raw || a->grad_dtype == STK_F32, "stk_optim_step_ex: reduced main gradients are fp32");
  if (a->n_local == 0 && !(a->lp_ptrs && a->lp_world > 1)) return STK_OK;
  const bool cross = a->lp_ptrs != nullptr && a->lp_world > 1;
  if (cross) {
    if (!c->comm_ready) return stk_fail(c, STK_ERR_STATE, "stk_optim_step (sharded) before stk_comm_connect");
    STK_POLL(c);
  }
  std::lock_guard<std::mutex> lk(c->mu);
  DeviceGuard g(c->device);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);

  OptimParams p{};
  p.master = a->master;
  p.m = a->exp_avg;
  p.v = a->exp_avg_sq;
  p.grad = a->grad;
  p.acc = a->grad_raw ? a->acc : nullptr;
  p.nvec = a->n_local / 8;
  p.lp_world = a->lp_ptrs ? a->lp_world : 0;
  p.lp_rank_skip = -1;
  // segments (vector units); the plain call is one segment at lp_offset
  bool pair_ok = true;
  if (a->n_seg == 0) {
    STK_REQUIRE(c, a->lp_offset % 8 == 0, "stk_optim_step_ex: lp_offset must be a multiple of 8");
    p.n_seg = 1;
    p.seg_local[0] = 0;
    p.seg_local[1] = (uint32_t)p.nvec;
    p.seg_global[0] = (uint32_t)(a->lp_offset / 8);
    pair_ok = (p.seg_global[0] % 2) == 0;
  } else {
    p.n_seg = a->n_seg;
    for (int k = 0; k <= a->n_seg; ++k) {
      STK_REQUIRE(c, a->seg_local[k] % 8 == 0, "stk_optim_step_ex: segment bounds must be multiples of 8");
      p.seg_local[k] = (uint32_t)(a->seg_local[k] / 8);
      if (k < a->n_seg) {
        STK_REQUIRE(c, a->seg_global[k] % 8 == 0, "stk_optim_step_ex: segment offsets must be multiples of 8");
        p.seg_global[k] = (uint32_t)(a->seg_global[k] / 8);
        pair_ok &= (p.seg_local[k] % 2) == 0 && (p.seg_global[k] % 2) == 0;
      }
    }
    STK_REQUIRE(c, p.seg_local[0] == 0 && p.seg_local[a->n_seg] == p.nvec, "stk_optim_step_ex: segments must tile [0, n_local)");
  }
  for (int r = 0; r < p.lp_world; ++r) {
    STK_REQUIRE(c, a->lp_ptrs[r] != nullptr, "stk_optim_step_ex: NULL lp pointer");
    p.lp.p[r] = a->lp_ptrs[r];
    if (a->lp_dtype == STK_F32 && p.n_seg == 1 &&
        static_cast<char*>(a->lp_ptrs[r]) + size_t(p.seg_global[0]) * 32 == reinterpret_cast<char*>(a->master))
      p.lp_rank_skip = r;
  }
  p.lp_mc = nullptr;
  if (cross && c->k2_ag_mc && a->lp_dtype != STK_F32) p.lp_mc = stk_mc_lookup(c, a->lp_ptrs[c->rank]);  // nullptr: not bound
  p.prof_ns = (cross && c->profiling) ? c->prof_ns_dev + 4 : nullptr;
  p.scaler = c->scaler_dev;
  p.pads = c->pads;
  p.rank = c->rank;
  p.world = c->world;
  p.cross_rank = cross ? 1 : 0;
  p.epoch = p.cross_rank ? ++c->blk_epoch : 0;
  p.kind = h->kind;
  p.clip_kind = h->clip_kind;
  p.clip_max_norm = (float)h->clip_max_norm;
  p.clip_value = (float)h->clip_value;
  p.grad_mul = (float)a->grad_mul;
  p.unscale = 0;
  p.n_groups = a->n_groups;
  fill_groups(p.g, h, a->hyper_ext, a->n_groups);
  p.any_mom = any_mom ? 1 : 0;
  p.n_ranges = a->n_ranges;
  p.range_end = a->range_end_vec;
  p.range_group = a->range_group;
  // the schedule-free scalars belong to the group (upstream keeps k per group), whatever the range table says
  p.range_bc = (a->n_ranges > 0 && !sf) ? reinterpret_cast<const float4*>(a->range_bc) : nullptr;
  p.group_bc = reinterpret_cast<const float4*>(a->group_bc);
  p.m2 = (ademamix || adan) ? a->exp_avg_slow : nullptr;
  p.m3 = adan ? m3 : nullptr;
  p.m_deferred = (ademamix && a->exp_avg && any_b1_zero) ? 1 : 0;
  if (rmsprop_tf) {
    p.m = any_rms_mom ? a->exp_avg : nullptr;
    p.m2 = any_centered ? a->exp_avg_slow : nullptr;
    p.m_deferred = (any_rms_mom && any_rms_no_mom) ? 1 : 0;
    p.m2_deferred = (any_centered && any_plain) ? 1 : 0;
    for (int gi = 0; gi < a->n_groups; ++gi) {   // the group's alpha and flags in the slots RMSpropTF does not use
      GroupHyperD& d = p.g[gi];
      d.rho = rt[gi].alpha;
      d.centered = rt[gi].centered != 0;
      d.decoupled = rt[gi].decoupled_decay != 0;
      d.buf_c = rt[gi].lr_in_momentum ? h[gi].lr : 1.0;
      d.upd_c = rt[gi].lr_in_momentum ? 1.0 : h[gi].lr;
    }
  }
  if (adan) {
    for (int gi = 0; gi < a->n_groups; ++gi) {   // beta3 and no_prox in the slots Adan does not use
      p.g[gi].rho = ad[gi].beta3;
      p.g[gi].decoupled = ad[gi].no_prox != 0;
    }
  }
  if (a->grad_raw) {
    // 1/loss_scale is applied when the scaler is live; the device flag decides (enabled), so no host read
    p.unscale = 1;
  }

  {
    static int pair_env = -1;   // STK_K2_PAIR=0: one vector per thread in the sharded step (16-byte peer stores, 3 blocks/SM)
    if (pair_env < 0) {
      const char* e = std::getenv("STK_K2_PAIR");
      pair_env = e ? std::atoi(e) : 1;
    }
    if (!pair_env) pair_ok = false;
  }
  cudaError_t err;
  const bool raw = a->grad_raw != 0;
  g_grid_nvec = cross ? (a->grid_n ? (a->grid_n + 7) / 8 : p.nvec) : 0;
  switch (h->kind) {
    case STK_OPT_ADAM: err = launch_optim<STK_OPT_ADAM>(c, p, a->lp_dtype, a->grad_dtype, raw, pair_ok, s); break;
    case STK_OPT_ADAMW: err = launch_optim<STK_OPT_ADAMW>(c, p, a->lp_dtype, a->grad_dtype, raw, pair_ok, s); break;
    case STK_OPT_NADAM: err = launch_optim<STK_OPT_NADAM>(c, p, a->lp_dtype, a->grad_dtype, raw, pair_ok, s); break;
    case STK_OPT_RADAM: err = launch_optim<STK_OPT_RADAM>(c, p, a->lp_dtype, a->grad_dtype, raw, pair_ok, s); break;
    case STK_OPT_ADAMAX: err = launch_optim<STK_OPT_ADAMAX>(c, p, a->lp_dtype, a->grad_dtype, raw, pair_ok, s); break;
    case STK_OPT_ADADELTA: err = launch_optim<STK_OPT_ADADELTA>(c, p, a->lp_dtype, a->grad_dtype, raw, pair_ok, s); break;
    case STK_OPT_RPROP: err = launch_optim<STK_OPT_RPROP>(c, p, a->lp_dtype, a->grad_dtype, raw, pair_ok, s); break;
    case STK_OPT_ASGD: err = launch_optim<STK_OPT_ASGD>(c, p, a->lp_dtype, a->grad_dtype, raw, pair_ok, s); break;
    case STK_OPT_LION: err = launch_optim<STK_OPT_LION>(c, p, a->lp_dtype, a->grad_dtype, raw, pair_ok, s); break;
    case STK_OPT_SF_ADAMW: err = launch_optim<STK_OPT_SF_ADAMW>(c, p, a->lp_dtype, a->grad_dtype, raw, pair_ok, s); break;
    case STK_OPT_SF_SGD: err = launch_optim<STK_OPT_SF_SGD>(c, p, a->lp_dtype, a->grad_dtype, raw, pair_ok, s); break;
    case STK_OPT_ADEMAMIX: err = launch_optim<STK_OPT_ADEMAMIX>(c, p, a->lp_dtype, a->grad_dtype, raw, pair_ok, s); break;
    case STK_OPT_RMSPROP_TF:
      err = launch_optim<STK_OPT_RMSPROP_TF>(c, p, a->lp_dtype, a->grad_dtype, raw, pair_ok, s);
      break;
    case STK_OPT_ADAN: err = launch_optim<STK_OPT_ADAN>(c, p, a->lp_dtype, a->grad_dtype, raw, pair_ok, s); break;
    default: err = launch_optim<STK_OPT_SGD>(c, p, a->lp_dtype, a->grad_dtype, raw, pair_ok, s); break;
  }
  if (err == cudaErrorNotSupported)
    return stk_fail(c, STK_ERR_UNSUPPORTED, "stk_optim_step_ex: this gradient dtype / parameter dtype pair has no raw route");
  if (err != cudaSuccess) return stk_fail(c, STK_ERR_CUDA, std::string("k_optim_step launch: ") + cudaGetErrorString(err));
  return STK_OK;
}

// What stk_optim_step_prologue, stk_ademamix_step_prologue and stk_adan_step_prologue share: the argument checks (`fn`
// names the entry point in their messages; `args_ok`: its own pointer arguments are set), the step-count bookkeeping
// fields, and the launch of one thread per range or per group.  `own(p)` checks and fills the rest of the parameters,
// returning STK_OK or the entry point's error.
template <typename Params, typename Own>
static int range_prologue(stk_ctx* c, const char* fn, bool args_ok, int n_groups, int n_ranges,
                          const uint8_t* range_group, int32_t* range_steps, float* bc, void (*kernel)(Params), Own own,
                          void* stream) {
  const std::string f(fn);
  STK_REQUIRE(c, c && args_ok && bc, f + ": NULL argument");
  STK_REQUIRE(c, n_groups >= 1 && n_groups <= STK_MAX_GROUPS, f + ": n_groups must be in [1, 8]");
  STK_REQUIRE(c, n_ranges >= 0, f + ": negative n_ranges");
  STK_REQUIRE(c, n_ranges == 0 || (range_group && range_steps), f + ": range arrays are NULL");
  STK_REQUIRE(c, (reinterpret_cast<uintptr_t>(bc) & 15) == 0, f + ": bc must be 16-byte aligned");
  Params p{};
  if (const int rc = own(p)) return rc;
  std::lock_guard<std::mutex> lk(c->mu);
  DeviceGuard g(c->device);
  p.n_groups = n_groups;
  p.n_ranges = n_ranges;
  p.range_group = range_group;
  p.range_steps = range_steps;
  p.bc = reinterpret_cast<float4*>(bc);
  p.scaler = c->scaler_dev;
  const int n = n_ranges > 0 ? n_ranges : n_groups;
  kernel<<<(n + 127) / 128, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  STK_CUDA(c, cudaGetLastError());
  return STK_OK;
}

extern "C" {

int stk_optim_step_ex(stk_ctx* c, const stk_optim_args_t* a, void* stream) {
  STK_REQUIRE(c, !(a && a->hyper && a->hyper->kind == STK_OPT_RMSPROP_TF),
              "stk_optim_step_ex: RMSPROP_TF takes its per-group hyper-parameters through stk_rmsprop_tf_step");
  STK_REQUIRE(c, !(a && a->hyper && a->hyper->kind == STK_OPT_ADAN),
              "stk_optim_step_ex: ADAN takes its per-group hyper-parameters and neg_pre_grad through stk_adan_step");
  return optim_step(c, a, nullptr, nullptr, nullptr, stream);
}

int stk_rmsprop_tf_step(stk_ctx* c, const stk_optim_args_t* a, const stk_rmsprop_tf_hyper_t* rt, void* stream) {
  STK_REQUIRE(c, c && a && a->hyper && rt, "stk_rmsprop_tf_step: NULL argument");
  STK_REQUIRE(c, a->hyper->kind == STK_OPT_RMSPROP_TF, "stk_rmsprop_tf_step: hyper->kind must be STK_OPT_RMSPROP_TF");
  return optim_step(c, a, rt, nullptr, nullptr, stream);
}

int stk_adan_step(stk_ctx* c, const stk_optim_args_t* a, const stk_adan_hyper_t* ad, float* neg_pre_grad, void* stream) {
  STK_REQUIRE(c, c && a && a->hyper && ad, "stk_adan_step: NULL argument");
  STK_REQUIRE(c, a->hyper->kind == STK_OPT_ADAN, "stk_adan_step: hyper->kind must be STK_OPT_ADAN");
  return optim_step(c, a, nullptr, ad, neg_pre_grad, stream);
}

int stk_optim_step(stk_ctx* c, const stk_optim_hyper_t* h, float* master, float* exp_avg, float* exp_avg_sq,
                   const float* grad, size_t n_local, void* const* lp_ptrs, int lp_world, int lp_dtype, size_t lp_offset,
                   void* stream) {
  STK_REQUIRE(c, c && h && master && grad, "stk_optim_step: NULL argument");
  stk_optim_args_t a{};
  a.hyper = h;
  a.n_groups = 1;
  a.master = master;
  a.exp_avg = exp_avg;
  a.exp_avg_sq = exp_avg_sq;
  a.grad = grad;
  a.grad_dtype = STK_F32;
  a.n_local = n_local;
  a.lp_ptrs = lp_ptrs;
  a.lp_world = lp_world;
  a.lp_dtype = lp_dtype;
  a.lp_offset = lp_offset;
  return stk_optim_step_ex(c, &a, stream);
}

int stk_optim_step_prologue(stk_ctx* c, const stk_optim_hyper_t* h, const stk_optim_hyper_ext_t* ext, int n_groups,
                            int n_ranges, const uint8_t* range_group, int32_t* range_steps, float* scalar_state, float* bc,
                            void* stream) {
  return range_prologue(c, "stk_optim_step_prologue", h, n_groups, n_ranges, range_group, range_steps, bc,
                        k_step_prologue, [&](StepPrologueParams& p) {
    STK_REQUIRE(c, (h->kind >= STK_OPT_ADAM && h->kind <= STK_OPT_SF_SGD) || h->kind == STK_OPT_RMSPROP_TF,
                "stk_optim_step_prologue: bad optimizer kind");
    STK_REQUIRE(c, scalar_state_width(h->kind) == 0 || scalar_state,
                "stk_optim_step_prologue: NAdam and ASGD need their scalar state");
    fill_groups(p.g, h, ext, n_groups);
    p.kind = h->kind;
    p.scalar_state = scalar_state;
    return (int)STK_OK;
  }, stream);
}

int stk_ademamix_step_prologue(stk_ctx* c, const stk_optim_hyper_t* h, const stk_ademamix_hyper_t* ah, int n_groups,
                               int n_ranges, const uint8_t* range_group, int32_t* range_steps, float* bc, void* stream) {
  return range_prologue(c, "stk_ademamix_step_prologue", h && ah, n_groups, n_ranges, range_group, range_steps, bc,
                        k_ademamix_prologue, [&](AdemamixPrologueParams& p) {
    for (int gi = 0; gi < n_groups; ++gi) {
      STK_REQUIRE(c, ah[gi].alpha_warmup >= 0 && ah[gi].beta3_warmup >= 0,
                  "stk_ademamix_step_prologue: warm-ups must be >= 0 (0: none)");
      p.beta1[gi] = h[gi].beta1;
      p.beta2[gi] = h[gi].beta2;
      p.a[gi] = ah[gi];
    }
    return (int)STK_OK;
  }, stream);
}

int stk_adan_step_prologue(stk_ctx* c, const stk_optim_hyper_t* h, const stk_adan_hyper_t* ah, int n_groups, int n_ranges,
                           const uint8_t* range_group, int32_t* range_steps, float* bc, void* stream) {
  return range_prologue(c, "stk_adan_step_prologue", h && ah, n_groups, n_ranges, range_group, range_steps, bc,
                        k_adan_prologue, [&](AdanPrologueParams& p) {
    for (int gi = 0; gi < n_groups; ++gi) {
      p.lr[gi] = h[gi].lr;
      p.beta1[gi] = h[gi].beta1;
      p.beta2[gi] = h[gi].beta2;
      p.a[gi] = ah[gi];
    }
    return (int)STK_OK;
  }, stream);
}

int stk_sf_step_prologue(stk_ctx* c, const stk_sf_hyper_t* h, int n_groups, double* group_state, float* bc, void* stream) {
  STK_REQUIRE(c, c && h && group_state && bc, "stk_sf_step_prologue: NULL argument");
  STK_REQUIRE(c, n_groups >= 1 && n_groups <= STK_MAX_GROUPS, "stk_sf_step_prologue: n_groups must be in [1, 8]");
  STK_REQUIRE(c, (reinterpret_cast<uintptr_t>(bc) & 15) == 0, "stk_sf_step_prologue: bc must be 16-byte aligned");
  for (int gi = 0; gi < n_groups; ++gi)
    STK_REQUIRE(c, h[gi].warmup_steps >= 0, "stk_sf_step_prologue: warmup_steps must be >= 0");
  std::lock_guard<std::mutex> lk(c->mu);
  DeviceGuard g(c->device);
  SfPrologueParams p{};
  for (int gi = 0; gi < n_groups; ++gi) p.g[gi] = h[gi];
  p.n_groups = n_groups;
  p.state = group_state;
  p.bc = reinterpret_cast<float4*>(bc);
  p.scaler = c->scaler_dev;
  k_sf_prologue<<<1, 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  STK_CUDA(c, cudaGetLastError());
  return STK_OK;
}

int stk_step_epilogue(stk_ctx* c, void* stream) {
  STK_REQUIRE(c, c != nullptr, "stk_step_epilogue: NULL ctx");
  STK_POLL(c);
  DeviceGuard g(c->device);
  k_step_epilogue<<<1, 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(c->scaler_dev, c->accum_dev);
  STK_CUDA(c, cudaGetLastError());
  return STK_OK;
}

}  // extern "C"
