// llq_policy.cu -- on-device forward of the PMC actor (include/llq_policy.h; SURVEY.md 8 row f2), sm_90a.
//
// One CTA (256 threads = 8 warps) owns a tile of M = 32 observation rows and walks the whole net with the activations in
// shared memory ([row][feature], padded so that the MMA A-fragment loads are conflict free).  The fully connected layers run
// on the tensor cores as 3xTF32 (`mma.sync.m16n8k8.tf32`, fp32 accumulate): every operand is split into a TF32 head and a
// remainder (truncation split) and the three significant products a_lo*b_hi + a_hi*b_lo + a_hi*b_hi are accumulated, which restores fp32-level
// accuracy (the 12 outputs are joint targets for the physics and the parity bar is 1e-4, so plain TF32 -- a 1e-3 perturbation that
// can also flip the discrete code -- is not an option).  The weights are re-ordered on the device (pmc_pack_kernel, at
// llq_policy_create and at every llq_policy_set_weights) into MMA B-fragment order, so a warp fetches the fragments of a k-step with one coalesced 8-byte load per lane and n-tile; they stream
// through L2 (1.4 MB per CTA) double-buffered in registers four k-steps ahead (LLQ_POLICY_KU).  An earlier version of this kernel
// did the same layers with fp32 FFMA (one output neuron per thread, 32 accumulators).
// The tile is 32 rows, not 128, on purpose: 4096 envs -> 128 CTAs = one wave over the H100's 132 SMs; a 128-row tile (one
// wgmma M = 64 pair per warpgroup) would leave 100 SMs idle at this batch.  The 32-code search, the 256 -> 1 value output and the
// Gaussian sampling stay on the CUDA cores.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>
#include <new>
#include <string>
#include <vector>
#include "../../include/llq.h"
#include "../../include/llq_policy.h"
#include "llq_philox.cuh"

#ifndef LLQ_POLICY_KU
#define LLQ_POLICY_KU 4      // k-steps of weight fragments per register buffer (two buffers)
#endif

namespace {

constexpr int M = 32, THREADS = 256;
constexpr int N_PROP = 135, N_FUT = 72, N_OBS = 207, H = 256, Z = 32, NCODE = 256, PE = 64, ZE = 32, NACT = 12;
constexpr int LDX = 212, LDH = 260;          // row strides (floats): stride/4 odd -> the 8 rows x 4 columns of an A fragment hit 32 banks
constexpr int ACT_NONE = 0, ACT_RELU = 1, ACT_TANH = 2;

struct Layer { const float2* w; const float* b; };   // B fragments [ktile][ntile][lane] = {W[8kt+t][8nt+g], W[8kt+t+4][8nt+g]}; bias padded
struct Weights {
  const float *prop_mean, *prop_std, *fut_mean, *fut_std;
  Layer v1, v2; const float* v3w; const float* v3b;
  Layer e1, e2, e3; const float* code;
  Layer pe, ze, d1, d2, d3;
  const float* logstd;
};

// x = hi + lo with hi = x truncated to TF32 (one LOP3) and lo = x - hi (exact in fp32, <= 13 significant bits).  The tensor
// core reads only the TF32 bits of an operand register, i.e. it truncates lo to 11 significant bits itself: the dropped part
// is <= 2^-21 |x|, the same order as the a_lo * b_lo product 3xTF32 leaves out.  (Truncation costs one LOP3
// per value where a rounding cvt.rna.tf32.f32 split costs several instructions: the splits must not fill the issue slots.)
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
  hi = __float_as_uint(x) & 0xffffe000u;
  lo = __float_as_uint(x - __uint_as_float(hi));
}

__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

template <int ACT>
__device__ __forceinline__ float activate(float v) {
  if (ACT == ACT_RELU) return fmaxf(v, 0.f);
  if (ACT == ACT_TANH) return tanhf(v);
  return v;
}

// out[m][n] = act(b[n] + sum_k A[m][k] W[k][n]) for the CTA's 32 rows; KT k-tiles of 8, NTILES n-tiles of 8.
// A warp owns MT m-tiles (of 16 rows) x NT n-tiles; warps beyond (2/MT) * (NTILES/NT) idle.  TRANSPOSE: out[n * M + m].
template <int KT, int NTILES, int MT, int NT, int ACT, bool TRANSPOSE>
__device__ __forceinline__ void mma_layer(const float* A, int lda, Layer L, float* out, int ldo) {
  constexpr int MG = 2 / MT, NG = NTILES / NT, KU = LLQ_POLICY_KU;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  if (warp >= MG * NG) return;
  const int m0 = (warp % MG) * MT * 16, nt0 = (warp / MG) * NT;
  float acc[MT][NT][4];
#pragma unroll
  for (int i = 0; i < NT; i++) {
    const float b0 = L.b[(nt0 + i) * 8 + 2 * t], b1 = L.b[(nt0 + i) * 8 + 2 * t + 1];
#pragma unroll
    for (int mi = 0; mi < MT; mi++) { acc[mi][i][0] = b0; acc[mi][i][1] = b1; acc[mi][i][2] = b0; acc[mi][i][3] = b1; }
  }
  const float2* wp = L.w + (size_t)nt0 * 32 + lane;
  float2 bc[KU][NT], bn[KU][NT];
#pragma unroll
  for (int u = 0; u < KU; u++)
#pragma unroll
    for (int i = 0; i < NT; i++) bc[u][i] = (u < KT) ? __ldg(wp + ((size_t)u * NTILES + i) * 32) : make_float2(0.f, 0.f);
#pragma unroll 1
  for (int kg = 0; kg < KT; kg += KU) {
#pragma unroll
    for (int u = 0; u < KU; u++)
#pragma unroll
      for (int i = 0; i < NT; i++)
        bn[u][i] = (kg + KU + u < KT) ? __ldg(wp + ((size_t)(kg + KU + u) * NTILES + i) * 32) : make_float2(0.f, 0.f);
#pragma unroll
    for (int u = 0; u < KU; u++) {
      const int kt = kg + u;
      if (kt < KT) {
        const float* ap = A + (m0 + g) * lda + kt * 8 + t;
        uint32_t ah[MT][4], al[MT][4];
#pragma unroll
        for (int mi = 0; mi < MT; mi++) {
          split_tf32(ap[(mi * 16) * lda], ah[mi][0], al[mi][0]);
          split_tf32(ap[(mi * 16 + 8) * lda], ah[mi][1], al[mi][1]);
          split_tf32(ap[(mi * 16) * lda + 4], ah[mi][2], al[mi][2]);
          split_tf32(ap[(mi * 16 + 8) * lda + 4], ah[mi][3], al[mi][3]);
        }
        uint32_t bh[NT][2], bl[NT][2];
#pragma unroll
        for (int i = 0; i < NT; i++) {
          split_tf32(bc[u][i].x, bh[i][0], bl[i][0]);
          split_tf32(bc[u][i].y, bh[i][1], bl[i][1]);
        }
        // the three products of one accumulator are MT*NT instructions apart (small terms first), so no MMA waits on its predecessor
#pragma unroll
        for (int i = 0; i < NT; i++)
#pragma unroll
          for (int mi = 0; mi < MT; mi++) mma_tf32(acc[mi][i], al[mi], bh[i][0], bh[i][1]);
#pragma unroll
        for (int i = 0; i < NT; i++)
#pragma unroll
          for (int mi = 0; mi < MT; mi++) mma_tf32(acc[mi][i], ah[mi], bl[i][0], bl[i][1]);
#pragma unroll
        for (int i = 0; i < NT; i++)
#pragma unroll
          for (int mi = 0; mi < MT; mi++) mma_tf32(acc[mi][i], ah[mi], bh[i][0], bh[i][1]);
      }
    }
#pragma unroll
    for (int u = 0; u < KU; u++)
#pragma unroll
      for (int i = 0; i < NT; i++) bc[u][i] = bn[u][i];
  }
#pragma unroll
  for (int mi = 0; mi < MT; mi++)
#pragma unroll
    for (int i = 0; i < NT; i++) {
      const int row = m0 + mi * 16 + g, col = (nt0 + i) * 8 + 2 * t;
      const float v0 = activate<ACT>(acc[mi][i][0]), v1 = activate<ACT>(acc[mi][i][1]);
      const float v2 = activate<ACT>(acc[mi][i][2]), v3 = activate<ACT>(acc[mi][i][3]);
      if (!TRANSPOSE) {
        *reinterpret_cast<float2*>(out + row * ldo + col) = make_float2(v0, v1);
        *reinterpret_cast<float2*>(out + (row + 8) * ldo + col) = make_float2(v2, v3);
      } else {
        out[col * M + row] = v0; out[(col + 1) * M + row] = v1;
        out[col * M + row + 8] = v2; out[(col + 1) * M + row + 8] = v3;
      }
    }
}

__global__ void __launch_bounds__(THREADS) pmc_policy_kernel(const float* __restrict__ obs, long long ld, int n, Weights w,
                                                             float* __restrict__ act, int* __restrict__ codes,
                                                             float* __restrict__ values, float* __restrict__ neglogp,
                                                             unsigned long long seed, unsigned long long counter, long long out_ld, long long row_gid0) {
  extern __shared__ __align__(16) float sm[];
  float* X = sm;                       // [M][LDX]  normalised observation, column 207 = 0
  float* P = X + M * LDX;              // [M][LDH]
  float* Q = P + M * LDH;              // [M][LDH]
  __shared__ int s_code[M];
  const int row0 = blockIdx.x * M;
  const int tid = threadIdx.x;
  // ---- normalise + clip (pmc_net.py:130-137), coalesced along the observation row
  for (int idx = tid; idx < M * (N_OBS + 1); idx += THREADS) {
    const int m = idx / (N_OBS + 1), k = idx - m * (N_OBS + 1);
    float v = 0.f;
    if (k < N_OBS) {
      const int row = row0 + m < n ? row0 + m : n - 1;
      const float mean = k < N_PROP ? w.prop_mean[k] : w.fut_mean[k - N_PROP];
      const float sd = k < N_PROP ? w.prop_std[k] : w.fut_std[k - N_PROP];
      v = fminf(fmaxf((obs[(size_t)row * ld + k] - mean) / (sd + 1e-8f), -5.0f), 5.0f);
    }
    X[m * LDX + k] = v;
  }
  __syncthreads();
  // ---- value head 207 -> 256 -> 256 -> 1, tanh (pmc_net.py:139-144); only when the caller wants it
  if (values != nullptr) {
    mma_layer<26, 32, 2, 4, ACT_TANH, false>(X, LDX, w.v1, P, LDH);
    __syncthreads();
    mma_layer<32, 32, 2, 4, ACT_TANH, false>(P, LDH, w.v2, Q, LDH);
    __syncthreads();
    const int warp = tid >> 5, lane = tid & 31;
    for (int m = warp; m < M; m += THREADS / 32) {
      float s = 0.f;
      for (int k = lane; k < H; k += 32) s = fmaf(Q[m * LDH + k], w.v3w[k], s);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0 && row0 + m < n) values[(size_t)(row0 + m) * out_ld] = s + w.v3b[0];
    }
    __syncthreads();
  }
  // ---- VQ encoder 207 -> 256 -> 256 -> 32 (pmc_net.py:33-45)
  mma_layer<26, 32, 2, 4, ACT_RELU, false>(X, LDX, w.e1, P, LDH);
  __syncthreads();
  mma_layer<32, 32, 2, 4, ACT_RELU, false>(P, LDH, w.e2, Q, LDH);
  __syncthreads();
  mma_layer<32, 4, 1, 1, ACT_NONE, true>(Q, LDH, w.e3, P, 0);           // z transposed: P[k * M + m]
  __syncthreads();
  // ---- nearest code: thread c owns code c, squared distance to all M rows; then per-row argmin (first index wins ties)
  {
    float d[M];
#pragma unroll
    for (int m = 0; m < M; m++) d[m] = 0.f;
    for (int k = 0; k < Z; k++) {
      const float c = w.code[k * NCODE + tid];
      const float4* z4 = reinterpret_cast<const float4*>(P + k * M);
#pragma unroll
      for (int m4 = 0; m4 < M / 4; m4++) {
        const float4 z = z4[m4];
        float t;
        t = z.x - c; d[4 * m4] = fmaf(t, t, d[4 * m4]);
        t = z.y - c; d[4 * m4 + 1] = fmaf(t, t, d[4 * m4 + 1]);
        t = z.z - c; d[4 * m4 + 2] = fmaf(t, t, d[4 * m4 + 2]);
        t = z.w - c; d[4 * m4 + 3] = fmaf(t, t, d[4 * m4 + 3]);
      }
    }
#pragma unroll
    for (int m = 0; m < M; m++) Q[m * LDH + tid] = d[m];   // dist[m][c]: consecutive codes in consecutive banks
  }
  __syncthreads();
  {
    const int warp = tid >> 5, lane = tid & 31;
    for (int m = warp; m < M; m += THREADS / 32) {
      float best = 3.4e38f; int bi = 0;
      for (int c = lane; c < NCODE; c += 32) {
        const float v = Q[m * LDH + c];
        if (v < best) { best = v; bi = c; }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ob < best || (ob == best && oi < bi)) { best = ob; bi = oi; }
      }
      if (lane == 0) { s_code[m] = bi; if (codes && row0 + m < n) codes[row0 + m] = bi; }
    }
  }
  __syncthreads();
  // quantised code -> Q[m][0..31]; prop_embed 135 -> 64 into P[m][0..63]; z_embed 32 -> 32 into P[m][64..95] (pmc_net.py:99-106)
  for (int idx = tid; idx < Z * M; idx += THREADS) {
    const int m = idx / Z, k = idx - m * Z;
    Q[m * LDH + k] = w.code[k * NCODE + s_code[m]];
  }
  __syncthreads();
  mma_layer<17, 8, 2, 1, ACT_RELU, false>(X, LDX, w.pe, P, LDH);          // weight rows >= 135 are zero: X[:, 135] (future[0]) drops out
  mma_layer<4, 4, 1, 1, ACT_RELU, false>(Q, LDH, w.ze, P + PE, LDH);
  __syncthreads();
  // ---- decoder 96 -> 256 -> 256 -> 12 (pmc_net.py:47-58)
  mma_layer<12, 32, 2, 4, ACT_RELU, false>(P, LDH, w.d1, Q, LDH);
  __syncthreads();
  mma_layer<32, 32, 2, 4, ACT_RELU, false>(Q, LDH, w.d2, P, LDH);
  __syncthreads();
  mma_layer<32, 2, 1, 1, ACT_NONE, false>(P, LDH, w.d3, Q, LDH);          // mean in Q[m][0..11]
  __syncthreads();
  // ---- output: the mean (agent.step(argmax=True)) or a sample of the diagonal Gaussian head with its -log p (pmc_net.py:107-113)
  if (tid < M && row0 + tid < n) {
    const int row = row0 + tid;
    const float* mean = Q + tid * LDH;
    float* a = act + (size_t)row * NACT;
    if (neglogp == nullptr) {
#pragma unroll
      for (int j = 0; j < NACT; j++) a[j] = mean[j];
    } else {
      float eps[NACT];
#pragma unroll
      for (int q4 = 0; q4 < NACT / 4; q4++) {
        const uint4 r = philox4x32(make_uint4((uint32_t)(row_gid0 + row), (uint32_t)q4, (uint32_t)counter, (uint32_t)(counter >> 32)),
                                   make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
        const float u0 = ((float)r.x + 0.5f) * 2.3283064365386963e-10f, u1 = (float)r.y * 2.3283064365386963e-10f;
        const float u2 = ((float)r.z + 0.5f) * 2.3283064365386963e-10f, u3 = (float)r.w * 2.3283064365386963e-10f;
        const float r0 = sqrtf(-2.0f * logf(fminf(u0, 0.99999994f))), r1 = sqrtf(-2.0f * logf(fminf(u2, 0.99999994f)));
        float s0, c0, s1, c1;
        sincosf(6.283185307179586f * u1, &s0, &c0);
        sincosf(6.283185307179586f * u3, &s1, &c1);
        eps[4 * q4] = r0 * c0; eps[4 * q4 + 1] = r0 * s0; eps[4 * q4 + 2] = r1 * c1; eps[4 * q4 + 3] = r1 * s1;
      }
      float nl = 0.5f * NACT * 1.8378770664093453f;          // 0.5 n log(2 pi)
#pragma unroll
      for (int j = 0; j < NACT; j++) {
        const float ls = w.logstd[j];
        a[j] = fmaf(expf(ls), eps[j], mean[j]);
        nl += 0.5f * eps[j] * eps[j] + ls;
      }
      neglogp[(size_t)row * out_ld] = nl;
    }
  }
}

// ---- the weight image: the 28 arrays of the blob re-ordered for pmc_policy_kernel.  Plain arrays are copied, every fully connected
// layer becomes its B fragments ([ktile][ntile][lane] float2 = {W[8kt+t][8nt+g], W[8kt+t+4][8nt+g]}, zero outside [K) x [N)) and its
// bias padded to the n-tiles, every piece starts on a 16-byte boundary and the gaps are zero.  The host computes only where the pieces
// go (image_layout); pmc_pack_kernel writes the image from the raw blob in device memory, at create and at every refresh.
enum PieceKind { P_PLAIN = 0, P_FRAG = 1, P_BIAS = 2 };
struct Piece { int kind, src, dst, K, N; };   // P_PLAIN: K floats; P_FRAG: W[K][N]; P_BIAS: b[N]; all offsets in floats
constexpr int kPieces = 28;                    // one per array of the blob
struct Layout { Piece p[kPieces]; int total; };

// piece blockIdx.y covers the image floats [dst, next piece's dst) (the last one up to total); every float of the image is written
__global__ void __launch_bounds__(THREADS) pmc_pack_kernel(const float* __restrict__ raw, float* __restrict__ img, Layout L) {
  const int pi = blockIdx.y;
  const Piece P = L.p[pi];
  const int end = pi + 1 < kPieces ? L.p[pi + 1].dst : L.total;
  const int NT = (P.N + 7) >> 3;
  for (int j = blockIdx.x * THREADS + threadIdx.x; P.dst + j < end; j += gridDim.x * THREADS) {
    float v = 0.f;
    if (P.kind == P_PLAIN) {
      if (j < P.K) v = raw[P.src + j];
    } else if (P.kind == P_BIAS) {
      if (j < P.N) v = raw[P.src + j];
    } else {
      const int tile = j >> 6, lane = (j >> 1) & 31, kt = tile / NT, nt = tile - kt * NT;
      const int k = kt * 8 + (lane & 3) + 4 * (j & 1), nn = nt * 8 + (lane >> 2);
      if (k < P.K && nn < P.N) v = raw[P.src + k * P.N + nn];
    }
    img[P.dst + j] = v;
  }
}

// where the pieces of the 28 arrays (include/llq_policy.h) go in the image: piece i holds array i; a zero total flags a mismatch
Layout image_layout() {
  Layout L{};
  int src = 0, dst = 0, i = 0;
  auto align = [&]() { dst = (dst + 3) & ~3; };
  auto plain = [&](int cnt) { align(); L.p[i++] = Piece{P_PLAIN, src, dst, cnt, 0}; src += cnt; dst += cnt; };
  auto layer = [&](int K, int N) {
    const int KT = (K + 7) / 8, NT = (N + 7) / 8;
    align(); L.p[i++] = Piece{P_FRAG, src, dst, K, N}; src += K * N; dst += KT * NT * 64;
    align(); L.p[i++] = Piece{P_BIAS, src, dst, 0, N}; src += N; dst += NT * 8;
  };
  plain(N_PROP); plain(N_PROP); plain(N_FUT); plain(N_FUT);
  layer(N_OBS, H); layer(H, H); plain(H); plain(1);
  layer(N_OBS, H); layer(H, H); layer(H, Z); plain(Z * NCODE);
  layer(N_PROP, PE); layer(Z, ZE); layer(PE + ZE, H); layer(H, H); layer(H, NACT);
  plain(NACT);
  L.total = dst;
  return (i == kPieces && src == LLQ_POLICY_N_WEIGHTS) ? L : Layout{};
}

thread_local std::string g_err;
int fail(int code, const char* msg) { g_err = msg; return code; }

constexpr int SMEM_BYTES = (int)(sizeof(float) * (M * LDX + 2 * M * LDH));
constexpr int kPackBlocks = 32;                // CTAs per piece: 8192 threads over at most 65 536 floats

}  // namespace

// d_raw: the raw blob of the last create / host refresh (the pack kernel's source); h_stage: pinned host staging of host refreshes, its
// copy to d_raw followed by ev_stage
struct llq_policy {
  int device; float* d_w; float* d_raw; Layout layout; Weights w;
  float* h_stage = nullptr; cudaEvent_t ev_stage = nullptr; bool staged = false;
};

namespace {

int pack(llq_policy* h, const float* d_src, cudaStream_t stream) {
  pmc_pack_kernel<<<dim3(kPackBlocks, kPieces), THREADS, 0, stream>>>(d_src, h->d_w, h->layout);
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? LLQ_OK : fail(LLQ_ECUDA, cudaGetErrorString(e));
}

void release(llq_policy* h) {
  cudaFree(h->d_w); cudaFree(h->d_raw);
  if (h->h_stage) cudaFreeHost(h->h_stage);
  if (h->ev_stage) cudaEventDestroy(h->ev_stage);
  delete h;
}

}  // namespace

extern "C" {

const char* llq_policy_last_error(void) { return g_err.c_str(); }

int llq_policy_create(const float* weights, int64_t n_weights, int32_t device, llq_policy_handle* out) {
  if (!weights || !out) return fail(LLQ_EINVAL, "null argument");
  if (n_weights != LLQ_POLICY_N_WEIGHTS) return fail(LLQ_EINVAL, "weight blob has the wrong length (include/llq_policy.h)");
  const Layout layout = image_layout();
  if (layout.total == 0) return fail(LLQ_EINVAL, "internal: weight layout mismatch");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(LLQ_ECUDA, "no CUDA device visible (no CPU fallback)");
  if (device < 0 || device >= ndev) return fail(LLQ_EINVAL, "device ordinal out of range");
  llq_policy* h = new (std::nothrow) llq_policy();
  if (!h) return fail(LLQ_ENOMEM, "out of memory");
  h->device = device; h->d_w = nullptr; h->d_raw = nullptr; h->layout = layout;
  cudaSetDevice(device);
  // the raw blob goes up as it is, the pack kernel writes the image from it; the create returns once the image is complete
  if (cudaMalloc(&h->d_w, sizeof(float) * layout.total) != cudaSuccess || cudaMalloc(&h->d_raw, sizeof(float) * LLQ_POLICY_N_WEIGHTS) != cudaSuccess) {
    release(h); return fail(LLQ_ECUDA, "cudaMalloc failed");
  }
  if (cudaMemcpy(h->d_raw, weights, sizeof(float) * LLQ_POLICY_N_WEIGHTS, cudaMemcpyHostToDevice) != cudaSuccess) {
    release(h); return fail(LLQ_ECUDA, "weight upload failed");
  }
  if (pack(h, h->d_raw, 0) != LLQ_OK) { release(h); return LLQ_ECUDA; }
  if (cudaStreamSynchronize(0) != cudaSuccess) { release(h); return fail(LLQ_ECUDA, "weight pack failed"); }
  const float* D = h->d_w;
  const Piece* p = layout.p;
  auto L = [&](int i) { Layer l; l.w = reinterpret_cast<const float2*>(D + p[i].dst); l.b = D + p[i + 1].dst; return l; };
  Weights& w = h->w;
  w.prop_mean = D + p[0].dst; w.prop_std = D + p[1].dst; w.fut_mean = D + p[2].dst; w.fut_std = D + p[3].dst;
  w.v1 = L(4); w.v2 = L(6); w.v3w = D + p[8].dst; w.v3b = D + p[9].dst;
  w.e1 = L(10); w.e2 = L(12); w.e3 = L(14); w.code = D + p[16].dst;
  w.pe = L(17); w.ze = L(19); w.d1 = L(21); w.d2 = L(23); w.d3 = L(25);
  w.logstd = D + p[27].dst;
  if (cudaFuncSetAttribute(pmc_policy_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES) != cudaSuccess) {
    release(h); return fail(LLQ_ECUDA, "cannot reserve shared memory for the policy kernel");
  }
  *out = h;
  return LLQ_OK;
}

int llq_policy_set_weights(llq_policy_handle h, const float* weights, int64_t n_weights, int32_t on_device, void* stream) {
  if (!h || !weights) return fail(LLQ_EINVAL, "null argument");
  if (n_weights != LLQ_POLICY_N_WEIGHTS) return fail(LLQ_EINVAL, "weight blob has the wrong length (include/llq_policy.h)");
  if (on_device != 0 && on_device != 1) return fail(LLQ_EINVAL, "on_device must be 0 (host memory) or 1 (device memory)");
  if (cudaSetDevice(h->device) != cudaSuccess) return fail(LLQ_ECUDA, "cudaSetDevice failed");
  const cudaStream_t s = (cudaStream_t)stream;
  const size_t bytes = sizeof(float) * LLQ_POLICY_N_WEIGHTS;
  if (on_device) {
    cudaPointerAttributes a{};
    if (cudaPointerGetAttributes(&a, weights) != cudaSuccess || a.type != cudaMemoryTypeDevice || a.device != h->device) {
      cudaGetLastError();
      return fail(LLQ_EINVAL, "on_device = 1 needs device memory on the handle's device");
    }
    return pack(h, weights, s);                // straight from the caller's blob
  }
  if (!h->h_stage && (cudaHostAlloc(&h->h_stage, bytes, cudaHostAllocDefault) != cudaSuccess ||
                      cudaEventCreateWithFlags(&h->ev_stage, cudaEventDisableTiming) != cudaSuccess))
    return fail(LLQ_ECUDA, "cannot allocate the pinned staging buffer");
  // the previous host refresh's copy must have left the staging buffer before it is overwritten: the only host wait
  if (h->staged && cudaEventSynchronize(h->ev_stage) != cudaSuccess) return fail(LLQ_ECUDA, "staging event failed");
  memcpy(h->h_stage, weights, bytes);
  if (cudaMemcpyAsync(h->d_raw, h->h_stage, bytes, cudaMemcpyHostToDevice, s) != cudaSuccess ||
      cudaEventRecord(h->ev_stage, s) != cudaSuccess)
    return fail(LLQ_ECUDA, "weight upload failed");
  h->staged = true;
  return pack(h, h->d_raw, s);
}

int llq_policy_destroy(llq_policy_handle h) {
  if (!h) return LLQ_OK;
  cudaSetDevice(h->device);
  release(h);
  return LLQ_OK;
}

int llq_policy_forward_rec(llq_policy_handle h, const float* d_obs, int64_t obs_ld, int32_t n, float* d_actions, int32_t* d_codes,
                           float* d_values, float* d_neglogp, int64_t out_ld, uint64_t seed, uint64_t counter, int64_t row_gid0, void* stream) {
  if (!h || !d_obs || !d_actions || n <= 0 || obs_ld < N_OBS || out_ld < 1) return fail(LLQ_EINVAL, "bad arguments");
  cudaSetDevice(h->device);
  pmc_policy_kernel<<<(n + M - 1) / M, THREADS, SMEM_BYTES, (cudaStream_t)stream>>>(d_obs, (long long)obs_ld, n, h->w, d_actions, d_codes,
                                                                                      d_values, d_neglogp, seed, counter, (long long)out_ld, (long long)row_gid0);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(LLQ_ECUDA, cudaGetErrorString(e));
  return LLQ_OK;
}

int llq_policy_forward_ex(llq_policy_handle h, const float* d_obs, int64_t obs_ld, int32_t n, float* d_actions, int32_t* d_codes,
                          float* d_values, float* d_neglogp, uint64_t seed, uint64_t counter, void* stream) {
  return llq_policy_forward_rec(h, d_obs, obs_ld, n, d_actions, d_codes, d_values, d_neglogp, 1, seed, counter, 0, stream);
}

int llq_policy_forward(llq_policy_handle h, const float* d_obs, int64_t obs_ld, int32_t n, float* d_actions, int32_t* d_codes, void* stream) {
  return llq_policy_forward_ex(h, d_obs, obs_ld, n, d_actions, d_codes, nullptr, nullptr, 0, 0, stream);
}

}  // extern "C"
