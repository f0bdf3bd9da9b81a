/*
 * stoke_b200.h -- C ABI of libstoke_b200.so (hand-written sm_90a kernels for the post-backward gradient path of
 * fidelity/stoke).  Plain C: opaque context, raw device pointers, sizes, and a cudaStream_t passed as void*.  No torch
 * types.  Every function returns 0 on success or a negative stk_status; the message is available through
 * stk_last_error().  No function synchronises the device unless its comment says so.  A context may be used from any
 * host thread (internally locked); all launches go to the stream the caller passes.
 *
 * What each entry point replaces in the reference (paths relative to /root/reference):
 *
 *   stk_ctx_create / stk_comm_*     process-group bring-up            stoke/distributed.py:491-538 (DistributedDDP)
 *   stk_mem_*                        DDP bucket storage (torch Reducer buckets, NCCL buffers)  stoke/extensions.py:207-215
 *   stk_grad_accumulate              local accumulation under no_sync  stoke/distributed.py:648-669, stoke/stoke.py:978-984
 *   stk_grad_reduce                  DDP bucket copy-in + all-reduce + copy-out (stoke/extensions.py:207-215), fused with
 *                                    GradScaler.unscale_ (stoke/fp16.py:180-183,222-225) and the norm / inf reductions of
 *                                    clip_grad_norm_ (stoke/fp16.py:233); reduce-scatter flavour = fairscale SDDP/OSS
 *                                    reduce-to-owner (stoke/extensions.py:277-285)
 *   stk_optim_step                   clip_grad_norm_/clip_grad_value_ scaling (stoke/fp16.py:184,233), scaler.step gate +
 *                                    optimizer.step() (stoke/fp16.py:298,805), OSS shard step + parameter broadcast
 *                                    (stoke/extensions.py:136-141 -> fairscale OSS.step)
 *   stk_step_epilogue                scaler.update() (stoke/fp16.py:806) + zero_grad bookkeeping (stoke/utils.py:83-106)
 *   stk_loss_sync                    detach_and_sync_loss: item + barrier + all_reduce + item  stoke/distributed.py:619-646
 *   stk_barrier                      torch.distributed.barrier()      stoke/distributed.py:673
 *   stk_bcast                        DDP init param sync / per-forward buffer broadcast (broadcast_buffers=True,
 *                                    stoke/configs.py:182)
 *   stk_randperm / stk_argsort_u32 / stk_sampler_*    BucketedDistributedSampler  stoke/data.py:156-266, 380-498
 *   stk_state_*                      one scaler / step-counter / norm state per optimizer (the reference keeps them per
 *                                    GradScaler / per optimizer object: stoke/fp16.py:733-806, stoke/extensions.py:53-78)
 *   stk_multicast_try_bind           NCCL's NVLS transport under DDP (stoke/extensions.py:207-215): an NVSwitch multicast
 *                                    mapping of a peer-visible buffer, used by the multimem flavour of stk_grad_reduce
 *   stk_grad_norm                    the two reduction passes of clip_grad_norm_ + GradScaler.unscale_'s inf test
 *                                    (stoke/fp16.py:180-183, 233) when there is no cross-rank reduce to fuse them into
 *   stk_grad_scale                   clip_grad_norm_'s scaling pass / clip_grad_value_ (stoke/fp16.py:184, 233) for the
 *                                    stock-optimizer route (any torch.optim class, stoke/extensions.py:53-78)
 *   stk_loss_sync_begin/_wait        detach_and_sync_loss without the per-micro-step host synchronisation
 *   stk_optim_step_prologue          the per-step scalars of the kinds after SGD; torch's per-parameter `state[p]["step"]`
 *                                    (torch/optim/adam.py: a parameter whose grad is None is not stepped and keeps its own
 *                                    count) for models with sometimes-unused parameters; NAdam's `state[p]["mu_product"]`
 *                                    (torch/optim/nadam.py) and ASGD's `state[p]["eta"]` / `["mu"]` (torch/optim/asgd.py)
 *                                    without `.item()`
 *   stk_adafactor_plan / _step       torch.optim.Adafactor's step (torch/optim/_adafactor.py _single_tensor_adafactor) plus
 *                                    the clip and the GradScaler.step gate, without its two .item() per parameter
 *   stk_layerwise_step               the step of the LAMB / LARS classes of stoke_b200.optim (per-parameter trust ratios;
 *                                    torch.optim has neither), plus the clip and the GradScaler.step gate
 */
#ifndef STOKE_B200_H
#define STOKE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define STK_MAX_WORLD 8
#define STK_IPC_HANDLE_BYTES 64

typedef struct stk_ctx stk_ctx;

typedef enum {
  STK_OK = 0,
  STK_ERR_INVALID = -1,   /* bad argument */
  STK_ERR_CUDA = -2,      /* a CUDA runtime call failed (no device, OOM, launch failure, ...) */
  STK_ERR_STATE = -3,     /* call order violated (e.g. reduce before comm connect) */
  STK_ERR_PEER = -4,      /* a peer did not arrive within the spin bound (dead or out-of-order rank) */
  STK_ERR_UNSUPPORTED = -5
} stk_status;

typedef enum { STK_F32 = 0, STK_BF16 = 1, STK_F16 = 2 } stk_dtype;

typedef enum {
  STK_REDUCE_ALL = 0,     /* all-reduce: owner reduces its shard and pushes the result to every rank */
  STK_REDUCE_SCATTER = 1  /* reduce-scatter: owner keeps its shard (ZeRO-1 / OSS) */
} stk_reduce_mode;

typedef enum { STK_NORM_NONE = 0, STK_NORM_L2 = 1, STK_NORM_INF = 2, STK_NORM_P = 3 } stk_norm_kind;
typedef enum { STK_CLIP_NONE = 0, STK_CLIP_NORM = 1, STK_CLIP_VALUE = 2 } stk_clip_kind;
typedef enum {
  STK_OPT_ADAM = 0, STK_OPT_ADAMW = 1, STK_OPT_SGD = 2,
  STK_OPT_NADAM = 3,   /* torch.optim.NAdam (torch/optim/nadam.py, _single_tensor_nadam) */
  STK_OPT_RADAM = 4,   /* torch.optim.RAdam (torch/optim/radam.py, _single_tensor_radam) */
  STK_OPT_ADAMAX = 5,  /* torch.optim.Adamax (torch/optim/adamax.py, _single_tensor_adamax); exp_avg_sq holds exp_inf */
  STK_OPT_ADADELTA = 6,  /* torch.optim.Adadelta (_single_tensor_adadelta); exp_avg = square_avg, exp_avg_sq = acc_delta */
  STK_OPT_RPROP = 7,   /* torch.optim.Rprop (_single_tensor_rprop); exp_avg = prev, exp_avg_sq = step_size */
  STK_OPT_ASGD = 8     /* torch.optim.ASGD (_single_tensor_asgd); exp_avg = ax, no exp_avg_sq */
} stk_optim_kind;

/* flags of stk_grad_reduce */
#define STK_RF_FINAL 1u        /* last bucket of this optimizer step: finish norm / found_inf (cross-rank exchange) */
#define STK_RF_ZERO_INPUT 2u   /* zero the local gradient bucket after it has been consumed (the accumulator is left as it
                                  is: the next stk_grad_accumulate with first != 0 overwrites it) */
#define STK_RF_UNSCALE 4u      /* multiply by 1/loss_scale (device scaler state) and test for inf/nan */

typedef struct {
  int sm_major, sm_minor, sm_count;
  int rank, world, device;
  int peer_access;        /* 1 if every peer's memory is mapped */
  int multicast;          /* 1 if the device reports CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED and the driver's VMM / multicast
                             entry points resolved (whether a given buffer is bound: stk_multicast_try_bind) */
  size_t hbm_bytes;
} stk_caps_t;

/* device-resident loss-scaler / step state (one per context); mirrors torch.amp.GradScaler's state_dict */
typedef struct {
  float scale;            /* current loss scale */
  float growth_factor, backoff_factor;
  int32_t growth_interval;
  int32_t growth_tracker;
  int32_t enabled;        /* 0: scale is fixed at 1 and never updated */
  int32_t found_inf;      /* result of the last finished reduce (all ranks agree) */
  float grad_norm;        /* total gradient norm of the last finished reduce (before clipping) */
  int64_t opt_steps;      /* optimizer steps actually applied (not skipped) */
  int64_t skipped_steps;
} stk_scaler_state_t;

typedef struct {
  int kind;               /* stk_optim_kind */
  double lr, beta1, beta2, eps, weight_decay;   /* Adam / AdamW / NAdam / RAdam / Adamax */
  double momentum, dampening;                   /* SGD */
  int nesterov;
  int maximize;
  int clip_kind;          /* stk_clip_kind */
  double clip_max_norm;   /* STK_CLIP_NORM: max_norm (norm kind / p were given to stk_grad_reduce) */
  double clip_value;      /* STK_CLIP_VALUE */
} stk_optim_hyper_t;

/* Per-group hyper-parameters of the kinds after SGD that stk_optim_hyper_t has no field for (one entry per group, same
 * order as the stk_optim_hyper_t array).  A NULL array means every field is 0.  stk_optim_hyper_t's lr, eps, weight_decay
 * and maximize apply to every kind that has them (Adadelta: lr, eps, weight_decay; Rprop: lr; ASGD: lr, weight_decay). */
typedef struct {
  double momentum_decay;        /* NAdam: momentum_decay (psi): mu_t = beta1 (1 - 0.5 * 0.96^(t psi)), torch/optim/nadam.py */
  int decoupled_weight_decay;   /* NAdam / RAdam: 1 = param *= 1 - lr wd before the update (AdamW-style); 0 = L2, grad += wd param */
  double rho;                   /* Adadelta: rho */
  double etaminus, etaplus;     /* Rprop: etas */
  double step_size_min, step_size_max;  /* Rprop: step_sizes */
  double lambd, alpha, t0;      /* ASGD */
} stk_optim_hyper_ext_t;

/* ---- library / context -------------------------------------------------------------------------------------------- */
int stk_version(void);
const char* stk_last_error(stk_ctx* ctx); /* ctx may be NULL: last error of the calling thread */

int stk_ctx_create(int rank, int world, int device, unsigned flags, stk_ctx** out);
int stk_ctx_destroy(stk_ctx* ctx);
int stk_caps(stk_ctx* ctx, stk_caps_t* out);

/* ---- peer-visible device memory; the 64-byte handles are exchanged by the caller ------------------------------------
 * Two back ends behind the same calls (STK_OPT_MEM_MODE / env STK_MEM=ipc|vmm, default vmm when world > 1 and the driver
 * supports it): "vmm" = cuMemCreate + POSIX file-descriptor export (the descriptor travels over a unix socket served by the
 * owning context) -- required for NVLS multicast; "ipc" = cudaMalloc + cudaIpc*.  All ranks must use the same mode. */
int stk_mem_alloc_shared(stk_ctx* ctx, size_t bytes, void** local_ptr, unsigned char handle_out[STK_IPC_HANDLE_BYTES]);
/* handles: world * 64 bytes in rank order; peer_ptrs_out[rank] == local_ptr.  In vmm mode this also imports the multicast
 * object rank 0 created for the buffer (if any) and adds this rank's device to it. */
int stk_mem_open_peers(stk_ctx* ctx, void* local_ptr, const unsigned char* handles, void** peer_ptrs_out);
int stk_mem_free_shared(stk_ctx* ctx, void* local_ptr);
/* Binds the buffer's memory to its multicast object and maps it: *mc_ptr_out is an address whose loads/stores address the
 * same offset of EVERY rank's buffer (multimem.* instructions).  Collective: call on every rank after every rank has returned
 * from stk_mem_open_peers (caller barrier), and barrier again before the first use.  Returns STK_ERR_UNSUPPORTED (and leaves
 * the buffer fully usable through its peer pointers) when the device, driver or buffer has no multicast support.
 * stk_multicast_release undoes a bind (used when some other rank failed to bind). */
int stk_multicast_try_bind(stk_ctx* ctx, void* local_ptr, void** mc_ptr_out);
int stk_multicast_release(stk_ctx* ctx, void* local_ptr);

/* signal pads (flags + scalar slots) used by every cross-rank kernel: two-phase like the buffers above */
int stk_comm_local(stk_ctx* ctx, unsigned char handle_out[STK_IPC_HANDLE_BYTES]);
int stk_comm_connect(stk_ctx* ctx, const unsigned char* handles);
/* copies the device error word to the host (synchronises `stream`); returns STK_ERR_PEER if a spin bound was hit */
int stk_comm_check(stk_ctx* ctx, void* stream);
/* same verdict without synchronising: reads the error word's mirror in mapped host memory (a kernel that gave up on a peer
 * writes it).  Every cross-rank entry point calls this first, so after a peer failure the next call returns STK_ERR_PEER. */
int stk_comm_poll(stk_ctx* ctx);

/* tuning knobs.  STK_OPT_K1_ALGO: how the cross-rank K1 brings the peers' 16-bit gradients into the SM -- 0 = 16-byte
 * register loads, 1 = bulk-async copies (TMA engine) staged through shared memory (default; +10..20 % bus bandwidth).  Same
 * results either way; fp32 gradients and launches with a local accumulator always take flavour 0.
 * Also settable at context creation through the environment variable STK_K1_ALGO=ldg|bulk. */
#define STK_OPT_K1_ALGO 1
/* 2 = multimem (NVLS): multimem.ld_reduce of the owned shard + multimem.st of the result; taken when the gradient and
 *     output buffers are multicast-bound and there is no local accumulator, otherwise the call falls back to 1 / 0.
 *     16-bit sums are rounded to the input type by the switch (fp32 accumulation inside it) -- NCCL's NVLS numerics.
 * STK_OPT_MEM_MODE: 0 = ipc, 1 = vmm (see stk_mem_alloc_shared).  STK_OPT_K1_MAX_BLOCKS: grid bound of the cross-rank
 * K1 (default: one block per SM); smaller grids leave SMs to a concurrently running backward. */
#define STK_OPT_MEM_MODE 2
#define STK_OPT_K1_MAX_BLOCKS 3
#define STK_OPT_COOP_LAUNCH 4   /* 1 (default): cross-rank kernels use cooperative launches (co-residency enforced) */
#define STK_OPT_NVLS_MAX_BLOCKS 5 /* grid bound of the multimem flavour alone (0: same as STK_OPT_K1_MAX_BLOCKS) */
#define STK_OPT_K2_AG_MC 6      /* 1: the sharded step publishes its shard with multimem.st when the parameter buffer is bound */
int stk_option_set(stk_ctx* ctx, int key, int value);
int stk_option_get(stk_ctx* ctx, int key, int* value);

/* launch timing for bench.py's roofline: when enabled, K1 (kind 0), K2 (kind 1) and the accumulate kernel (kind 2) are
 * bracketed by CUDA events on the launch stream; stk_profile_read synchronises those events, returns the summed
 * duration and the launch count since the last read, and clears the list. */
int stk_profile_enable(stk_ctx* ctx, int on);
int stk_profile_read(stk_ctx* ctx, int kind, double* ms_total, int* launches);
/* cross-rank K1 only: time between its start and end barriers (the NVLink data phase) taken with the device timer by block 0 --
 * excludes the wait for the slowest rank to arrive, which host-side events include; ms_zero_tail (may be NULL) receives
 * the time block 0 then spent zeroing its part of the local bucket (HBM work).  Synchronises `stream`. */
int stk_profile_read_k1_device(stk_ctx* ctx, double* ms_total, int* launches, double* ms_zero_tail, void* stream);
/* the same for the sharded optimizer step (cross-rank K2): time between its start and end barriers = local update + the
 * parameter all-gather, without the wait for the slowest rank to arrive.  Synchronises `stream`. */
int stk_profile_read_k2_device(stk_ctx* ctx, double* ms_total, int* launches, void* stream);

/* ---- scaler / step state ------------------------------------------------------------------------------------------- */
/* One device-resident state (loss scaler, found_inf, grad_norm, step counters, per-step norm accumulators) per optimizer.
 * State 0 exists from stk_ctx_create.  stk_state_select makes `id` the state that stk_scaler_*, stk_grad_reduce,
 * stk_grad_norm, stk_grad_scale, stk_optim_step* and stk_step_epilogue read and write until the next select. */
int stk_state_create(stk_ctx* ctx, int* id_out);
int stk_state_select(stk_ctx* ctx, int id);
int stk_state_destroy(stk_ctx* ctx, int id);
int stk_scaler_set(stk_ctx* ctx, const stk_scaler_state_t* st, void* stream);
int stk_scaler_get(stk_ctx* ctx, stk_scaler_state_t* st, void* stream); /* synchronises `stream` */
void* stk_scaler_scale_ptr(stk_ctx* ctx); /* device float*: the live loss scale (for scaler.scale(loss)) */

/* ---- K1: gradient path --------------------------------------------------------------------------------------------- */
/* acc[i] (+)= float(grad[i]); optionally zero grad.  Local, HBM-bound.  first != 0 overwrites acc. */
int stk_grad_accumulate(stk_ctx* ctx, void* grad, int grad_dtype, float* acc, size_t n, int first, int zero_grad,
                        void* stream);

/* main[i] = (sum_r (grad_r[i] [+ acc_r[i]])) * mul * (1/scale)   for i in the shard this rank owns (all i if world==1),
 * written to every rank (STK_REDUCE_ALL) or kept locally (STK_REDUCE_SCATTER); accumulates the norm partial and the
 * inf/nan flag; with STK_RF_FINAL finishes them across ranks into the scaler state.
 *   grad_ptrs / acc_ptrs / out_ptrs: `world` device pointers in rank order (peer mappings); acc_ptrs may be NULL.
 *   n: elements in the bucket (multiple of 8);  mul: e.g. 1/world;  norm_kind / norm_p: which norm to accumulate. */
int stk_grad_reduce(stk_ctx* ctx, int mode, void* const* grad_ptrs, int grad_dtype, float* const* acc_ptrs,
                    void* const* out_ptrs, int out_dtype, size_t n, double mul, int norm_kind, double norm_p,
                    unsigned flags, void* stream);

/* Norm / inf pass without a reduce (world == 1, or gradients that were reduced elsewhere): accumulates the norm partial and
 * the inf/nan flag of x[i] = (float(grad[i]) [+ acc[i]]) * mul * (1/scale) over [0, n) into the selected state and, with
 * STK_RF_FINAL, finishes them (grad_norm, found_inf).  Reads grad once, writes nothing: stk_optim_step_ex then consumes the
 * raw bucket directly (no fp32 main-grad round trip through HBM).  Loads keep the bucket L2-resident for that second read. */
int stk_grad_norm(stk_ctx* ctx, const void* grad, int grad_dtype, const float* acc, size_t n, double mul, int norm_kind,
                  double norm_p, unsigned flags, void* stream);

/* In-place clip of already reduced fp32 gradients for the stock-optimizer route: grad[i] *= min(max_norm/(norm+1e-6), 1)
 * (STK_CLIP_NORM, norm from the selected state) or clamp (STK_CLIP_VALUE). */
int stk_grad_scale(stk_ctx* ctx, float* grad, size_t n, int clip_kind, double clip_max_norm, double clip_value, void* stream);

/* element range [begin, end) of the shard `rank` owns in a bucket of n elements (same partition the kernels use) */
int stk_shard_range(size_t n, int world, int rank, size_t* begin, size_t* end);

/* ---- K2: fused optimizer step (+ K3 parameter all-gather when sharded) ---------------------------------------------- */
/* Updates master/exp_avg/exp_avg_sq over [0, n_local) from grad (fp32, already reduced & unscaled); applies the clip
 * coefficient from the scaler state; skips everything if found_inf.  If lp_ptrs != NULL the updated parameters are also
 * written as lp_dtype to lp_ptrs[r] + lp_offset for r in [0, lp_world) (lp_world == 1: local low-precision copy;
 * lp_world == world: sharded step pushing its shard to every rank = parameter all-gather). */
int stk_optim_step(stk_ctx* ctx, const stk_optim_hyper_t* hyper, float* master, float* exp_avg, float* exp_avg_sq,
                   const float* grad, size_t n_local, void* const* lp_ptrs, int lp_world, int lp_dtype, size_t lp_offset,
                   void* stream);

/* Extended form.  Everything stk_optim_step does, plus:
 *  - raw gradient source (grad_raw = 1): `grad` is the local model-dtype bucket (+ optional fp32 accumulator), scaled by
 *    grad_mul and 1/loss_scale inside the kernel and ZEROED after it has been read (also on a skipped step); pairs with
 *    stk_grad_norm -- the world == 1 route: 2 + 30 B/element instead of 8 + 30.
 *  - segments: the local state [0, n_local) is the concatenation of n_seg pieces; piece k covers local elements
 *    [seg_local[k], seg_local[k+1]) and global (flat-buffer) elements starting at seg_global[k].  lp_ptrs / raw grads /
 *    the range table are indexed globally.  n_seg = 0: one piece, global offset lp_offset (the plain call).
 *  - parameter groups and unused parameters: n_ranges > 0 gives a table over the GLOBAL flat index space; range j ends at
 *    element range_end[j] (ascending, device memory, multiples of 8) and uses hyper[range_group[j] & 0x7f]; bit 7 set = skip
 *    the range this step (parameter received no gradient: torch skips it, torch/optim/optimizer.py).  n_ranges = 0: hyper[0]
 *    everywhere.  With 32-byte peer stores (bf16 parameters, segments on 16-element boundaries) a thread handles two adjacent
 *    vectors and looks the range up once: ranges must then end on 16-element boundaries. */
#define STK_MAX_GROUPS 8
#define STK_MAX_SEGMENTS 64
typedef struct {
  const stk_optim_hyper_t* hyper;   /* n_groups entries (clip fields taken from hyper[0]) */
  int n_groups;
  float* master; float* exp_avg; float* exp_avg_sq;
  const void* grad; int grad_dtype;  /* STK_F32 reduced main grads (local indexing) | raw bucket (global indexing) */
  int grad_raw;
  const float* acc;                  /* raw route only: fp32 accumulator added to grad (global indexing), may be NULL */
  double grad_mul;                   /* raw route only */
  size_t n_local;
  void* const* lp_ptrs; int lp_world; int lp_dtype; size_t lp_offset;
  int n_seg; const size_t* seg_local; const size_t* seg_global;   /* host arrays: n_seg + 1 and n_seg entries */
  int n_ranges; const uint32_t* range_end_vec; const uint8_t* range_group;  /* DEVICE arrays; ends in units of 8 elements */
  size_t grid_n;   /* cross-rank (lp_world > 1) launches: the LARGEST n_local over the ranks, identical on every rank, so that
                      every rank launches the same grid (the block barriers pair block b with block b); 0: n_local */
  const float* range_bc;  /* DEVICE, 4 floats per RANGE written by stk_optim_step_prologue with n_ranges > 0: per-PARAMETER
                             step counts (torch keeps `step` per parameter, so a parameter that skipped some steps has its
                             own bias corrections); NULL: group_bc */
  const stk_optim_hyper_ext_t* hyper_ext;  /* n_groups entries or NULL (all zero): the extras of the kinds after SGD */
  const float* group_bc;  /* DEVICE, 4 floats per GROUP written by stk_optim_step_prologue with n_ranges = 0; used where
                             range_bc is NULL.  NULL: ADAM / ADAMW / SGD form the scalars of the optimizer-wide step
                             themselves.  Every kind after SGD needs group_bc or range_bc: their per-step scalars (NAdam's
                             and ASGD's come from scalar state that only the prologue advances) are formed once by the
                             prologue, not in every block.  ASGD takes no exp_avg_sq */
} stk_optim_args_t;
int stk_optim_step_ex(stk_ctx* ctx, const stk_optim_args_t* args, void* stream);
/* Step bookkeeping for every kind, including the per-entry scalar state of NAdam and ASGD (call it right before
 * stk_optim_step_ex, same stream).
 * n_ranges > 0: per range j: the scalars of step t = range_steps[j] + 1 with the group hyper[range_group[j] & 0x7f] go to
 *   bc[4j..4j+3] (pass bc as the step's range_bc), and unless the range is skipped this step (bit 7 of range_group[j]) or
 *   the selected state says found_inf, range_steps[j] and entry j's scalar state advance.
 * n_ranges = 0: per group g, with t = the selected state's optimizer-wide counter + 1: bc[4g..4g+3] (pass bc as the
 *   step's group_bc) and, unless found_inf, entry g's scalar state advances.  range_group and range_steps are not read.
 * The four floats per entry, computed in double from torch's python-scalar formulas and stored as fp32:
 *   ADAM / ADAMW: {lr / bc1, sqrt(bc2), t == 1, 0}
 *   NADAM:  {c_g, c_m, bc2, 0}: param += c_g grad / denom + c_m exp_avg / denom, denom = sqrt(exp_avg_sq / bc2) + eps,
 *           c_g = -lr (1 - mu_t) / (1 - P_t), c_m = -lr mu_{t+1} / (1 - P_t mu_{t+1}), P_t = fp32(P_{t-1} * fp32(mu_t))
 *           is the advanced mu_product (torch: mu_product *= mu, then .item())
 *   RADAM:  {c, rectified, 0, 0}: rho_t = rho_inf - 2 t beta2^t / bc2 > 5 -> rectified = 1,
 *           c = lr rect sqrt(bc2) / bc1, param -= c exp_avg / (sqrt(exp_avg_sq) + eps); else rectified = 0,
 *           c = lr / bc1, param -= c exp_avg
 *   ADAMAX: {lr / bc1, 0, 0, 0}: param -= (lr / bc1) exp_avg / exp_inf
 *   SGD, ADADELTA, RPROP: {0, 0, t == 1, 0}: SGD's first step seeds the momentum buffer with the gradient; Rprop's seeds
 *           step_size with the lr passed now (torch: full_like(p, lr) at the parameter's first step) and takes prev as 0;
 *           the exp_avg_sq buffer is not used then
 *   ASGD:   {-eta, 1 - lambd eta, mu, 0} with the STORED fp32 eta and mu (the lr and 1 at t == 1, torch's lazy
 *           initialisation): param = param (1 - lambd eta) - eta grad; ax = param if mu == 1 (ax not read), else
 *           ax + (param - ax) mu.  Then eta = lr / (1 + lambd lr t)^alpha and mu = 1 / max(1, t - t0), as fp32
 * with bc1 = 1 - beta1^t, bc2 = 1 - beta2^t.  The scalar state `scalar_state` (fp32, torch keeps it per parameter) holds per
 * range or per group: NADAM one float, mu_product (torch initialises it to 1); ASGD two floats, {eta, mu}.  It is read and
 * written only for those two kinds and may be NULL for the others; hyper_ext may be NULL (all zero).
 * All pointers but hyper / hyper_ext are device memory; bc must be 16-byte aligned. */
int stk_optim_step_prologue(stk_ctx* ctx, const stk_optim_hyper_t* hyper, const stk_optim_hyper_ext_t* hyper_ext,
                            int n_groups, int n_ranges, const uint8_t* range_group, int32_t* range_steps,
                            float* scalar_state, float* bc, void* stream);

/* scaler.update(), opt_steps/skipped_steps bookkeeping, reset of the per-step accumulators */
int stk_step_epilogue(stk_ctx* ctx, void* stream);

/* ---- Adafactor: fused step of torch.optim.Adafactor ------------------------------------------------------------------
 * Replaces torch/optim/_adafactor.py _single_tensor_adafactor (its per-parameter python loop with two .item() host
 * synchronisations), plus clip_grad_norm_ / clip_grad_value_'s scaling and GradScaler.step's inf gate, like stk_optim_step.
 * Per parameter with a gradient, t = its own step count after the increment:
 *   b2hat = t^beta2_decay, rho = min(lr, 1/sqrt(t)), alpha = max(eps2, ||w|| / sqrt(numel)) * rho   (norm BEFORE decay)
 *   w *= 1 - lr * weight_decay                                             (weight_decay != 0)
 *   dim >= 2: row_var = lerp(row_var, mean_c g^2, b2hat), col_var = lerp(col_var, mean_r g^2, b2hat) over the last two dims
 *             (leading dims are a batch), v = row_var[r] col_var[c] / clamp_min(mean_r row_var, eps1)
 *   dim <= 1: variance = lerp(variance, g^2, b2hat), v = variance
 *   u = g rsqrt(clamp_min(v, eps1^2)),  w += (-alpha / max(1, ||u|| / (sqrt(numel) d))) u
 * with python's max / min (a NaN norm gives eps2 and 1) and eps1 "None" = fp32 epsilon (the masters are fp32).
 * Deterministic: every sum adds in an order fixed by the shapes (per-block / per-chunk partials folded in index order by a
 * finisher), no floating-point atomics.  Nothing is synchronised; the launches go to `stream` in order. */
typedef struct {
  uint64_t offset;        /* first element of the parameter in the flat master / gradient / lp buffers */
  uint64_t state;         /* first element of its state in the state buffer */
  int32_t numel;          /* 1 .. 2^31 - 1 */
  int32_t factored;       /* 1 (dim >= 2): row_var [B*R] then col_var [B*C] at `state`, torch's contiguous [..., R, 1] and
                             [..., 1, C]; 0 (dim <= 1): variance [numel] */
  int32_t size[4];        /* logical sizes (B0, B1, R, C), left-padded with 1; B = B0 * B1 */
  int32_t stride[4];      /* element strides of those dims in the flat buffers; the parameter must be dense (any order) */
  /* filled by stk_adafactor_plan */
  int32_t contiguous, tile0, b0, pad_;
  int64_t line0, out0, rm0;
} stk_adafactor_param_t;

typedef struct {          /* totals of a plan (filled by stk_adafactor_plan) */
  int32_t n_params, n_tiles, n_b, pad_;
  int64_t n_line, n_out, n_rm;
  size_t workspace_bytes; /* device workspace stk_adafactor_step needs (no initialisation) */
} stk_adafactor_plan_t;

typedef struct {          /* one per parameter group */
  double lr, beta2_decay, eps1, eps2, d, weight_decay;
  int eps1_none;          /* 1: eps=(None, eps2): fp32 epsilon */
  int maximize;
} stk_adafactor_hyper_t;

typedef struct {
  const stk_adafactor_hyper_t* hyper; int n_groups;   /* host array, <= STK_MAX_GROUPS */
  int clip_kind; double clip_max_norm, clip_value;
  const stk_adafactor_param_t* params;  /* DEVICE copy of the planned table */
  const stk_adafactor_plan_t* plan;     /* host */
  const uint8_t* param_group;  /* DEVICE, one per parameter: group index, bit 7 = no gradient this step (not stepped) */
  int32_t* steps;              /* DEVICE, one per parameter: steps taken; advanced here unless skipped or found_inf */
  float* master;               /* fp32 masters (flat indexing) */
  float* state;                /* fp32 state buffer */
  void* workspace;             /* plan->workspace_bytes, 16-byte aligned */
  const void* grad; int grad_dtype; int grad_raw;  /* raw = 1: model-dtype bucket (bf16 | f32) scaled by grad_mul and
                                                      1/loss_scale, ZEROED after the step (also when skipped);
                                                      raw = 0: fp32 reduced main gradients */
  const float* acc; double grad_mul;  /* raw route: optional fp32 accumulator, multiplier */
  void* lp; int lp_dtype;      /* low-precision parameter copy written after the update (bf16 | f32), or NULL */
} stk_adafactor_args_t;

/* Validates `params_host[0..n)` (offset, state, numel, factored, size, stride filled by the caller) and fills their plan
 * fields and the totals.  Host only. */
int stk_adafactor_plan(stk_adafactor_param_t* params_host, int n_params, stk_adafactor_plan_t* plan_out);
/* One Adafactor step: eight stream-ordered launches (||w||^2 partials, per-parameter scalars and step counts, row / column
 * sums of g^2, their lerp, row means, ||u||^2 partials, the per-parameter coefficient, the update).  Reads the selected
 * scaler state (found_inf skips every parameter and leaves state and counts unchanged; the raw bucket is still zeroed). */
int stk_adafactor_step(stk_ctx* ctx, const stk_adafactor_args_t* args, void* stream);

/* ---- LAMB / LARS: layer-wise adaptive steps (stoke_b200.optim.LAMB / LARS) --------------------------------------------
 * The large-batch optimizers of BERT (LAMB) and ResNet-50 (LARS): an element-wise update scaled per parameter by a trust
 * ratio formed from two whole-parameter norms, plus clip_grad_norm_ / clip_grad_value_'s scaling and GradScaler.step's
 * inf gate, like stk_optim_step.  Per parameter with a gradient, g the gradient after unscale, accumulation and clip,
 * t = its own step count after the increment, adapt = weight_decay != 0 || always_adapt:
 *   LAMB: m = lerp(m, g, 1 - beta1);  v = v beta2 + (1 - beta2) g^2
 *         bc1, bc2 = 1 - beta1^t, 1 - beta2^t (double; 1 without bias_correction)
 *         r = (m / bc1) / (sqrt(v / bc2) + eps) + wd w
 *         trust = adapt && ||w|| > 0 && ||r|| > 0 ? ||w|| / ||r|| : 1          (w before this step's update)
 *         w -= lr (trust r)
 *   LARS: trust = adapt && ||w|| > 0 && ||g|| > 0 ? tc ||w|| / (||g|| + wd ||w|| + eps) : 1   (g before weight decay)
 *         adapt: g = (g + wd w) trust
 *         momentum != 0: buf = t == 1 ? g : buf momentum + (1 - dampening) g;  g = nesterov ? g + momentum buf : buf
 *         w -= lr g
 * A NaN norm fails the comparisons (trust 1), as torch.where does.  Three stream-ordered launches: a tile pass (per-tile
 * partial sums of w^2 and r^2 or g^2; LAMB also updates m, v and zeroes the raw bucket), a per-parameter fold (trust
 * ratio, step count), the update (fp32 master, low-precision copy; LARS: momentum buffer and bucket zeroing).  LAMB's
 * update recomputes r from the stored m, v and w with the same fp32 operations as the tile pass, so the r it applies is
 * the r whose norm it took.  Deterministic: every sum adds in an order fixed by the shapes, no floating-point atomics.
 * found_inf skips every parameter and a set bit 7 of its group byte skips one: master, state and count are left as they
 * are (the raw bucket is still zeroed).  Nothing is synchronised. */
#define STK_LW_TILE 8192   /* elements per tile of the tile passes */
typedef enum { STK_LW_LAMB = 0, STK_LW_LARS = 1 } stk_layerwise_kind;

typedef struct {          /* one per parameter */
  uint64_t offset;        /* first element in the flat master / gradient / state / lp buffers: a multiple of 16 */
  int32_t numel;          /* 0 .. 2^31 - 1; the elements after numel up to the next parameter are padding, left as they are */
  int32_t tile0;          /* first tile: the sum of ceil(numel / STK_LW_TILE) over the parameters before it */
} stk_layerwise_param_t;

typedef struct {          /* one per parameter group */
  double lr;
  double beta1, beta2;    /* LAMB */
  double eps, weight_decay;
  double momentum, dampening, trust_coefficient;  /* LARS */
  int bias_correction;    /* LAMB */
  int nesterov;           /* LARS */
  int always_adapt;       /* 1: the trust ratio also when weight_decay == 0 */
  int pad_;
} stk_layerwise_hyper_t;

typedef struct {
  int kind;                                           /* stk_layerwise_kind */
  const stk_layerwise_hyper_t* hyper; int n_groups;   /* host array, <= STK_MAX_GROUPS */
  int clip_kind; double clip_max_norm, clip_value;
  const stk_layerwise_param_t* params;  /* DEVICE table, ascending offsets */
  int n_params, n_tiles;                /* n_tiles: the sum of ceil(numel / STK_LW_TILE) */
  const uint8_t* param_group;  /* DEVICE, one per parameter: group index, bit 7 = no gradient this step (not stepped) */
  int32_t* steps;              /* DEVICE, one per parameter: steps taken; advanced here unless skipped or found_inf */
  float* master;               /* fp32 masters (flat indexing) */
  float* exp_avg;              /* LAMB: exp_avg; LARS: momentum_buffer (may be NULL when no group has momentum) */
  float* exp_avg_sq;           /* LAMB: exp_avg_sq; LARS: not used */
  void* workspace;             /* 16 n_params + 8 n_tiles bytes, 16-byte aligned, no initialisation */
  const void* grad; int grad_dtype; int grad_raw;  /* raw = 1: model-dtype bucket (bf16 | f32) scaled by grad_mul and
                                                      1/loss_scale, ZEROED after the step (also when skipped);
                                                      raw = 0: fp32 reduced main gradients */
  const float* acc; double grad_mul;  /* raw route: optional fp32 accumulator, multiplier */
  void* lp; int lp_dtype;      /* low-precision parameter copy written after the update (bf16 | f32), or NULL */
} stk_layerwise_args_t;
int stk_layerwise_step(stk_ctx* ctx, const stk_layerwise_args_t* args, void* stream);

/* ---- small collectives on the signal pads -------------------------------------------------------------------------- */
/* mean over ranks of *loss_dev (float32/bf16/f16 scalar) -> *out_host (pinned, mapped) ; synchronises `stream` */
int stk_loss_sync(stk_ctx* ctx, const void* loss_dev, int dtype, double* out_host, void* stream);
/* The same mean without the host synchronisation: _begin launches the kernel, which writes the mean to a slot of a pinned
 * ring and returns a ticket; _wait blocks until that launch has finished (no-op if it already has) and returns the value.
 * At most STK_LOSS_RING tickets may be outstanding (older slots are overwritten). */
#define STK_LOSS_RING 256
int stk_loss_sync_begin(stk_ctx* ctx, const void* loss_dev, int dtype, int64_t* ticket_out, void* stream);
int stk_loss_sync_wait(stk_ctx* ctx, int64_t ticket, double* out_host);
int stk_barrier(stk_ctx* ctx, void* stream);
/* every rank copies bytes from ptrs[root] to ptrs[rank] (peer pull) with start/end barriers */
int stk_bcast(stk_ctx* ctx, void* const* ptrs, size_t bytes, int root, void* stream);

/* ---- model forward ------------------------------------------------------------------------------------------------- */
/* The activation that follows the BatchNorm, as torch 2.11's CUDA kernels evaluate it on a bf16 input (fp32 opmath, one
 * rounding to bf16): relu (clamp_min(0)), silu (x / (1 + expf(-x))), hardswish (x * min(max(x + 3, 0), 6) * (1/6)),
 * relu6 (hardtanh(x, 0, 6) = clamp(x, 0, 6)).  relu and relu6 keep a NaN's bits. */
enum { STK_ACT_RELU = 0, STK_ACT_SILU = 1, STK_ACT_HARDSWISH = 2, STK_ACT_RELU6 = 3 };

/* Training-mode BatchNorm apply + optional residual add + activation `act` (STK_ACT_*) over a bf16 channels-last (NHWC)
 * tensor of `numel` elements and `channels` channels (multiple of 8, numel < 2^31, every pointer 16-byte aligned), from
 * statistics torch reduced (torch.batch_norm_update_stats: fp32 mean and biased var):
 *   out = act(bf16(bf16(weight * (x - mean) * invstd + bias) + residual)),  save_invstd[c] = rsqrtf(var[c] + eps)
 * with every intermediate rounded as the unfused torch ops round it (bit-identical to them).  residual may be NULL, and
 * must be NULL unless act is STK_ACT_RELU. */
int stk_bn_act_ex(stk_ctx* ctx, int act, const void* x, const void* residual, const float* mean, const float* var,
                  const void* weight, const void* bias, double eps, void* out, float* save_invstd, size_t numel,
                  size_t channels, void* stream);
/* stk_bn_act_ex with act = STK_ACT_RELU */
int stk_bn_act(stk_ctx* ctx, const void* x, const void* residual, const float* mean, const float* var, const void* weight,
               const void* bias, double eps, void* out, float* save_invstd, size_t numel, size_t channels, void* stream);

/* ---- model backward ------------------------------------------------------------------------------------------------ */
/* Backward of stk_bn_act_ex: the activation's backward followed by torch's training-mode BatchNorm backward, with the
 * coverage of stk_bn_act_ex (bf16 channels-last, channels % 8 == 0, numel < 2^31, every pointer 16-byte aligned).
 *   g = act_backward(grad, y);  sum_dy = sum g,  sum_dy_xmu = sum g * (x - mean)  (per channel over R = numel / channels)
 *   grad_bias = bf16(sum_dy),  grad_weight = bf16(sum_dy_xmu * invstd)
 *   grad_x = bf16(((g - sum_dy * n) - (x - mean) * (invstd * invstd * sum_dy_xmu * n)) * (weight * invstd)),  n = float(1.0 / R)
 * act_backward is torch's backward op of the activation, g rounded to bf16 as it rounds it:
 *   relu       threshold_backward(grad, out, 0) = !(out <= 0) ? grad : +0 (grad's bits kept)
 *   silu       silu_backward: s = 1 / (1 + expf(-y)); bf16(grad * s * fmaf(y, 1 - s, 1))
 *   hardswish  hardswish_backward: bf16(y <= -3 ? 0 : y < 3 ? grad * (y / 3 + 0.5) : grad)
 *   relu6      hardtanh_backward(grad, y, 0, 6): bf16(y <= 0 || y >= 6 ? 0 : grad)
 * out != NULL (STK_ACT_RELU only): a site with a residual; the mask comes from out and g is written to grad_residual.
 * out == NULL: y = bf16(weight * (x - mean) * invstd + bias) is recomputed, the formula stk_bn_act_ex applies (relu(y)
 * <= 0 iff y <= 0); grad_residual is unused.  grad_pre, when not NULL, receives g (2 B/element more; it exists so the
 * derivative can be tested apart from the sums, and must be NULL for STK_ACT_RELU, whose g keeps grad's bits or is +0).
 * grad_x may be NULL (no elementwise pass).
 * Order contract: the two sums add in the order of torch's batch_norm_backward_reduce_channels_last_kernel as launched by
 * flexible_launch_configs(R, channels, coop) with MAX_BLOCK_SIZE 512 (a function of R and channels only), so all four
 * outputs are bit-identical to act_backward + native_batch_norm_backward on channels-last bf16 inputs.
 * workspace: 2 * (1 + 128) * channels floats (the two sums, then per-block partials); no initialisation needed. */
int stk_bn_act_backward_ex(stk_ctx* ctx, int act, const void* grad, const void* x, const void* out, const float* mean,
                           const float* invstd, const void* weight, const void* bias, void* grad_x, void* grad_weight,
                           void* grad_bias, void* grad_residual, void* grad_pre, float* workspace, size_t numel,
                           size_t channels, void* stream);
/* stk_bn_act_backward_ex with act = STK_ACT_RELU and no grad_pre */
int stk_bn_act_backward(stk_ctx* ctx, const void* grad, const void* x, const void* out, const float* mean,
                        const float* invstd, const void* weight, const void* bias, void* grad_x, void* grad_weight,
                        void* grad_bias, void* grad_residual, float* workspace, size_t numel, size_t channels,
                        void* stream);

/* ---- sampler (stoke/data.py) ---------------------------------------------------------------------------------------- */
/* torch.randperm(n, generator=g) for each n in lens[0..k) drawn from ONE mt19937 seeded with `seed` (host, bit-exact
 * with torch's CPU generator); out receives the k permutations back to back as int32. */
int stk_randperm(uint64_t seed, const int64_t* lens, int k, int32_t* out_host);

typedef struct {
  int64_t n, buckets, batch_size, world, rank;
  int32_t drop_last, allow_bucket_overlap, shuffle;
  /* derived (filled by stk_sampler_plan) */
  int64_t slice_size, per_bucket, slices_per_bucket, rounded_per_bucket, rounded_per_replica;
  int64_t bucket_base, bucket_rem;   /* np.array_split: first bucket_rem buckets have bucket_base + 1 elements */
  int64_t n_bucket_batches, n_overlap_batches, n_batches;
  int32_t needs_padding;
} stk_sampler_plan_t;

/* Fills the derived fields; returns STK_ERR_INVALID with the reference's message for its three ValueError guards. */
int stk_sampler_plan(stk_sampler_plan_t* plan);
/* Positions (into the permuted bucket) of the padded last slice for a bucket of length `bucket_len`:
 * out[j], j in [0, slice_size), is the position that lands at offset j of the last slice (stoke/data.py:450-498). */
int stk_sampler_last_slice(const stk_sampler_plan_t* plan, int64_t bucket_len, int32_t* out_host);

/* stable argsort of u32 keys on the device (LSD radix, 8-bit digits): idx_out[i] = index of the i-th smallest key.
 * tmp must hold stk_argsort_tmp_bytes(n) bytes. */
size_t stk_argsort_tmp_bytes(size_t n);
int stk_argsort_u32(stk_ctx* ctx, const uint32_t* keys, size_t n, int64_t* idx_out, void* tmp, void* stream);

/* out[j] for j in [0, rounded_per_replica): this replica's epoch indices.
 *   sorted_idx: int64[n] (device); bucket_perm: int32[n] per-bucket permutations back to back (NULL if !shuffle);
 *   batch_perm: int32[n_batches] (NULL if !shuffle); last_slice: int32[2][slice_size] tables for bucket lengths
 *   bucket_base + 1 and bucket_base (NULL if !needs_padding). */
int stk_sampler_indices(stk_ctx* ctx, const stk_sampler_plan_t* plan, const int64_t* sorted_idx,
                        const int32_t* bucket_perm, const int32_t* batch_perm, const int32_t* last_slice,
                        int64_t* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* STOKE_B200_H */
