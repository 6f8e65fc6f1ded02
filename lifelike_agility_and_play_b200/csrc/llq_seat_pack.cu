// llq_seat_pack.cu -- the learner seat of a strategic-level trajectory slab (include/llq_policy.h, llq_seat_pack), sm_90a.
//
// SepmcRolloutWorker writes [T, 2P, 984] fp32 slabs: row 2p of each step is the learning robot of pair p (seat 0), row 2p + 1 its
// frozen opponent (seat 1).  The learner reads seat 0 only, and NCCL sends contiguous buffers, so the hand-over packs the seat-0 rows
// into a [T, P, 984] buffer first.  Output row r = t P + p comes from slab row t 2P + 2p = 2r: a 984-float record is 246 float4s and
// starts on a 16-byte boundary, so one thread moves one float4, vector i of the output coming from vector i + 246 * (i / 246) of the
// slab.  A bandwidth-bound copy (at T = 128, P = 4096: 2.06 GB read, 2.06 GB written); the loads are evict-first, since nothing
// reads the slab again before the worker rewrites it.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>
#include "../../include/llq.h"
#include "../../include/llq_policy.h"

namespace {

constexpr int kVec = LLQ_SEPMC_RECORD / 4;         // float4s per record (246)
constexpr int kThreads = 256;
constexpr long long kMaxVec = 2147483647LL * kThreads;    // gridDim.x <= 2^31 - 1
static_assert(LLQ_SEPMC_RECORD % 4 == 0, "a record must be whole float4s");

__global__ void __launch_bounds__(kThreads) seat_pack_kernel(const float4* __restrict__ slab, float4* __restrict__ out,
                                                             unsigned long long n_vec) {
  const unsigned long long i = (unsigned long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= n_vec) return;
  out[i] = __ldcs(slab + i + (i / kVec) * kVec);
}

thread_local std::string g_err;
int fail(int code, const char* msg) { g_err = msg; return code; }

}  // namespace

extern "C" {

const char* llq_seat_pack_last_error(void) { return g_err.c_str(); }

int llq_seat_pack(const float* d_slab, float* d_out, int64_t steps, int64_t pairs, void* stream) {
  if (!d_slab || !d_out) return fail(LLQ_EINVAL, "null pointer");
  if (((uintptr_t)d_slab | (uintptr_t)d_out) & 15) return fail(LLQ_EINVAL, "the slab and the output must be 16-byte aligned");
  if (steps <= 0 || pairs <= 0 || steps > kMaxVec / kVec / pairs) return fail(LLQ_EINVAL, "steps and pairs must be positive and fit one launch");
  const long long n_vec = steps * pairs * kVec;
  const uintptr_t s0 = (uintptr_t)d_slab, s1 = s0 + 32 * (uintptr_t)n_vec, o0 = (uintptr_t)d_out, o1 = o0 + 16 * (uintptr_t)n_vec;
  if (o0 < s1 && s0 < o1) return fail(LLQ_EINVAL, "the output overlaps the slab");
  cudaPointerAttributes a{}, b{};
  if (cudaPointerGetAttributes(&a, d_slab) != cudaSuccess || cudaPointerGetAttributes(&b, d_out) != cudaSuccess) {
    cudaGetLastError();
    return fail(LLQ_ECUDA, "cannot query the pointers (no CUDA device?)");
  }
  if (a.type != cudaMemoryTypeDevice || b.type != cudaMemoryTypeDevice || a.device != b.device)
    return fail(LLQ_EINVAL, "the slab and the output must be device memory on one device");
  int cur = -1;
  if (cudaGetDevice(&cur) != cudaSuccess || (cur != a.device && cudaSetDevice(a.device) != cudaSuccess)) return fail(LLQ_ECUDA, "cudaSetDevice failed");
  seat_pack_kernel<<<(unsigned)((n_vec + kThreads - 1) / kThreads), kThreads, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const float4*>(d_slab), reinterpret_cast<float4*>(d_out), (unsigned long long)n_vec);
  const cudaError_t e = cudaGetLastError();
  if (cur != a.device) cudaSetDevice(cur);
  return e == cudaSuccess ? LLQ_OK : fail(LLQ_ECUDA, cudaGetErrorString(e));
}

}  // extern "C"
