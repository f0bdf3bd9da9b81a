// weight_avg.cu -- the weight-average update (EMA / SWA of torch.optim.swa_utils.AveragedModel) over fp32 master weights:
// avg = master (mode 1) or avg = torch.lerp(avg, master, weight) (mode 2), one launch after every optimizer route's step.
// HBM bytes per element: 12 (lerp) or 8 (copy), 16-byte streaming accesses.  It is not folded into K2: carrying the lerp
// in K2's pass (38 instead of 30 + 12 B/element) costs registers and occupancy, and measured slower than this separate pass
// (DESIGN.md section 4).
#include "k1_common.cuh"

namespace stk {

// lerp_torch (k1_common.cuh): torch.lerp on fp32 with the contraction of torch's CUDA foreach-lerp kernel
template <int MODE>
__global__ void __launch_bounds__(256) k_weight_avg(float* __restrict__ avg, const float* __restrict__ master, size_t n4,
                                                    float w) {
  const size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  float4 m = ld_stream_f4(master + 4 * i);
  if (MODE == 2) {
    const float4 a = ld_stream_f4(avg + 4 * i);
    m = make_float4(lerp_torch(a.x, m.x, w), lerp_torch(a.y, m.y, w), lerp_torch(a.z, m.z, w), lerp_torch(a.w, m.w, w));
  }
  st_stream_f4(avg + 4 * i, m);
}

}  // namespace stk

using namespace stk;

extern "C" int stk_weight_avg(stk_ctx* c, float* avg, const float* master, size_t n, int mode, float weight, void* stream) {
  STK_REQUIRE(c, c && avg && master, "stk_weight_avg: NULL argument");
  STK_REQUIRE(c, mode == 1 || mode == 2, "stk_weight_avg: mode must be 1 (copy) or 2 (lerp)");
  STK_REQUIRE(c, n % 4 == 0, "stk_weight_avg: n must be a multiple of 4");
  STK_REQUIRE(c, ((reinterpret_cast<uintptr_t>(avg) | reinterpret_cast<uintptr_t>(master)) & 15) == 0,
              "stk_weight_avg: avg and master must be 16-byte aligned");
  if (n == 0) return STK_OK;
  DeviceGuard g(c->device);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const size_t n4 = n / 4;
  const unsigned grid = (unsigned)((n4 + 255) / 256);
  if (mode == 2) k_weight_avg<2><<<grid, 256, 0, s>>>(avg, master, n4, weight);
  else k_weight_avg<1><<<grid, 256, 0, s>>>(avg, master, n4, weight);
  STK_CUDA(c, cudaGetLastError());
  return STK_OK;
}
