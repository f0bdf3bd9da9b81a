// common.cuh -- device helpers shared by the stoke_b200 kernels (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/stoke_b200.h"

namespace stk {

constexpr int kMaxWorld = STK_MAX_WORLD;
constexpr int kMaxBlocks = 1024;
constexpr int kMaxReduceBlocks = 512;        // grid bound of the cross-rank K1 (one block per SM)             // upper bound on the grid of any cross-rank kernel (flag slots per peer)
constexpr uint64_t kDefaultSpinTimeoutNs = 600ull * 1000ull * 1000ull * 1000ull;  // 10 min (STK_SPIN_TIMEOUT_S): a dead peer becomes an error, not a hang

// ---- signal pad layout (one per rank, peer-mapped) ------------------------------------------------------------------
// All flags are monotonically increasing epochs written by the peer (st.release.sys) and polled locally
// (ld.acquire.sys); nothing is ever reset, so there is no reset race.
struct RankScalars {       // what a rank publishes about its shard at the end of a reduce
  float norm_partial;      // sum of squares / max / sum |g|^p over the shard
  uint32_t found_inf;
  uint32_t pad_[2];
};
struct SignalPad {
  uint32_t blk_flag[2][kMaxBlocks][kMaxWorld];  // [0]: start barrier, [1]: end barrier of block b, written by peer p
  uint32_t aux_flag[4][kMaxWorld];              // 0: (unused), 1: loss sync, 2: barrier kernel, 3: (unused)
  RankScalars blk_scal[kMaxWorld][kMaxReduceBlocks];  // [r][b]: norm partial / inf flag of rank r's K1 block b
  float loss_slot[2][kMaxWorld];                // double-buffered by call parity
  uint32_t error;                               // non-zero: a spin bound was hit on this rank
  // ---- local-only fields (peers never touch them) ----
  uint32_t pad0_;
  uint64_t timeout_ns;                          // spin bound of wait_flag
  uint32_t* host_err;                           // mapped pinned host word mirrored from `error` (polled by the host without a sync)
};

struct PeerPads {
  SignalPad* p[kMaxWorld];
};
struct PtrTable {
  void* p[kMaxWorld];
};

// ---- memory-model primitives -----------------------------------------------------------------------------------------
__device__ __forceinline__ void st_release_sys(uint32_t* addr, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* addr) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_sys_f32(float* addr, float v) {
  asm volatile("st.relaxed.sys.global.f32 [%0], %1;" ::"l"(addr), "f"(v) : "memory");
}
__device__ __forceinline__ void st_relaxed_sys_u32(uint32_t* addr, uint32_t v) {
  asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ float ld_relaxed_sys_f32(const float* addr) {
  float v;
  asm volatile("ld.relaxed.sys.global.f32 %0, [%1];" : "=f"(v) : "l"(addr) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_relaxed_sys_u32(const uint32_t* addr) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(addr) : "memory");
  return v;
}
__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// Wait until *flag >= epoch (epochs only grow).  Bounded: on timeout (or when this rank already failed) raises the local
// pad's error word AND its mirror in mapped host memory -- which every host entry point polls, so the next library call
// returns STK_ERR_PEER -- and returns false; callers abandon the kernel's data phase instead of consuming garbage.
__device__ __forceinline__ bool wait_flag(const uint32_t* flag, uint32_t epoch, SignalPad* mine) {
  uint32_t spins = 0;
  uint64_t t0 = 0;
  while ((int32_t)(ld_acquire_sys(flag) - epoch) < 0) {
    if ((++spins & 0x3ff) == 0) {
      uint64_t now = globaltimer_ns();
      if (t0 == 0) t0 = now;
      else if (now - t0 > mine->timeout_ns || ld_relaxed_sys_u32(&mine->error) != 0) {
        st_relaxed_sys_u32(&mine->error, 1u);
        if (mine->host_err) {
          *reinterpret_cast<volatile uint32_t*>(mine->host_err) = 1u;
          __threadfence_system();
        }
        return false;
      }
    }
  }
  return true;
}

// Block-to-block barrier across ranks: block b of every rank arrives, then block b of every rank proceeds.
// Call with all threads of the block.  `which` selects the start (0) or end (1) flag row.  Returns false (to every thread
// of the block) when a peer did not arrive within the spin bound.
__device__ __forceinline__ bool block_barrier_all_ranks(const PeerPads& pads, int rank, int world, int which,
                                                        uint32_t epoch) {
  __syncthreads();
  int ok = 1;
  if (threadIdx.x < (unsigned)world) {
    const int peer = threadIdx.x;
    __threadfence_system();
    st_release_sys(&pads.p[peer]->blk_flag[which][blockIdx.x][rank], epoch);
    ok = wait_flag(&pads.p[rank]->blk_flag[which][blockIdx.x][peer], epoch, pads.p[rank]) ? 1 : 0;
  }
  return __syncthreads_and(ok) != 0;
}

// ---- 16-byte vector access -------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 ld_stream16(const void* p) {  // streaming load, do not keep in L1
  uint4 v;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}
__device__ __forceinline__ void st_stream16(void* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w)
               : "memory");
}
__device__ __forceinline__ float4 ld_stream_f4(const float* p) {
  uint4 u = ld_stream16(p);
  return make_float4(__uint_as_float(u.x), __uint_as_float(u.y), __uint_as_float(u.z), __uint_as_float(u.w));
}
__device__ __forceinline__ void st_stream_f4(float* p, const float4& v) {
  st_stream16(p, make_uint4(__float_as_uint(v.x), __float_as_uint(v.y), __float_as_uint(v.z), __float_as_uint(v.w)));
}

// 32-byte accesses (one 8-element fp32 vector per thread).  sm_90 has no 256-bit global load / store: two adjacent
// 16-byte accesses, both issued before either result is used, so the thread's whole 32-byte sector is in flight at once.
struct f8 {
  float v[8];
};
__device__ __forceinline__ f8 ld_stream_f8(const float* p) {
  const uint4 a = ld_stream16(p), b = ld_stream16(p + 4);
  f8 r;
  r.v[0] = __uint_as_float(a.x); r.v[1] = __uint_as_float(a.y); r.v[2] = __uint_as_float(a.z); r.v[3] = __uint_as_float(a.w);
  r.v[4] = __uint_as_float(b.x); r.v[5] = __uint_as_float(b.y); r.v[6] = __uint_as_float(b.z); r.v[7] = __uint_as_float(b.w);
  return r;
}
__device__ __forceinline__ void st_stream_f8(float* p, const float (&v)[8]) {
  st_stream_f4(p, make_float4(v[0], v[1], v[2], v[3]));
  st_stream_f4(p + 4, make_float4(v[4], v[5], v[6], v[7]));
}

__device__ __forceinline__ float bf16lo(uint32_t u) { return __uint_as_float(u << 16); }
__device__ __forceinline__ float bf16hi(uint32_t u) { return __uint_as_float(u & 0xffff0000u); }
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float f16lo(uint32_t u) {
  return __half2float(__ushort_as_half((unsigned short)(u & 0xffffu)));
}
__device__ __forceinline__ float f16hi(uint32_t u) { return __half2float(__ushort_as_half((unsigned short)(u >> 16))); }
// the 8 bf16 or f16 values of one 16-byte vector, in memory order
template <int DT16>
__device__ __forceinline__ void unpack16(const uint4& u, float (&f)[8]) {
  static_assert(DT16 == STK_BF16 || DT16 == STK_F16, "unpack16 takes a 16-bit type");
  const uint32_t w4[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    f[2 * j] = (DT16 == STK_BF16) ? bf16lo(w4[j]) : f16lo(w4[j]);
    f[2 * j + 1] = (DT16 == STK_BF16) ? bf16hi(w4[j]) : f16hi(w4[j]);
  }
}

__device__ __forceinline__ bool finitef(float x) { return (__float_as_uint(x) & 0x7f800000u) != 0x7f800000u; }

// max that propagates NaN (max.NaN.f32, sm_80+), like torch's max / amax: fmaxf returns the non-NaN operand, which would
// turn the inf-norm of a gradient holding a NaN into a finite number.  Same result as fmaxf when neither input is NaN.
__device__ __forceinline__ float fmax_nan(float a, float b) {
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
// clamps that keep NaN, like torch.clamp (comparisons with NaN are false, so NaN falls through unchanged)
__device__ __forceinline__ float clamp_max_nan(float x, float hi) { return x > hi ? hi : x; }
__device__ __forceinline__ float clamp_nan(float x, float lo, float hi) { return x < lo ? lo : (x > hi ? hi : x); }

// ---- NVLS: multimem accesses on a multicast mapping (one address = the same offset in every rank's buffer; the NVSwitch
// reduces the W copies on a load and replicates a store).  SASS: LDGMC.E.ADD.* / STG on the multicast address. -------------
__device__ __forceinline__ uint4 mm_ld_reduce_bf16x8(const void* mc) {  // sum over ranks of 8 bf16, fp32 accumulation
  uint4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(mc)
               : "memory");
  return v;
}
__device__ __forceinline__ uint4 mm_ld_reduce_f16x8(const void* mc) {
  uint4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.f16x2 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(mc)
               : "memory");
  return v;
}
__device__ __forceinline__ float4 mm_ld_reduce_f32x4(const void* mc) {
  float4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(mc)
               : "memory");
  return v;
}
__device__ __forceinline__ void mm_st16(void* mc, const uint4& v) {  // 16 bytes replicated to every rank
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "f"(__uint_as_float(v.x)),
               "f"(__uint_as_float(v.y)), "f"(__uint_as_float(v.z)), "f"(__uint_as_float(v.w))
               : "memory");
}

// ---- block reductions (fixed tree -> deterministic) --------------------------------------------------------------------
template <bool kMax>
__device__ __forceinline__ float warp_reduce(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    float w = __shfl_xor_sync(0xffffffffu, v, o);
    v = kMax ? fmax_nan(v, w) : v + w;
  }
  return v;
}
template <bool kMax>
__device__ __forceinline__ float block_reduce(float v, float* smem /* >= 32 floats */) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = (blockDim.x + 31) >> 5;
  v = warp_reduce<kMax>(v);
  __syncthreads();
  if (lane == 0) smem[warp] = v;
  __syncthreads();
  if (warp == 0) {
    float x = lane < nwarp ? smem[lane] : (kMax ? 0.f : 0.f);
    x = warp_reduce<kMax>(x);
    if (lane == 0) smem[0] = x;
  }
  __syncthreads();
  float r = smem[0];
  return r;
}

}  // namespace stk
