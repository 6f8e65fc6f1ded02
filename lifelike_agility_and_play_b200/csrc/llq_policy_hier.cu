// On-device inference of the reference's environmental- and strategic-level policies (SURVEY.md 8 row f2; include/llq_policy.h).
//
//   networks/legged_robot/epmc_net/epmc_net.py:86-135   perception encoders (2-D / 1-D convolutions, SAME + ReLU) and their fusion
//   networks/legged_robot/epmc_net/epmc_net.py:138-177  mlc_encoder: prop 135 -> 64 | command 120 -> 64, concat -> 256 -> LSTM(32, layer norm)
//                                                       -> 256 logits -> argmax -> column of the primitive-level codebook
//   networks/legged_robot/sepmc_net/sepmc_net.py:122-146 hlc_encoder: prop | perception 88 -> 64 | game vector 29 -> 64 -> 64, concat 192 ->
//                                                       256 -> LSTM(32) -> heading angle; (cos, sin, commanded speed) = the mlc target
//   networks/legged_robot/pmc_net/pmc_net.py:99-112      llc: the frozen primitive-level decoder
// The LSTM is `tpolicies`' layer-norm LSTM (absent from the reference tree), restated as in lifelike_agility_and_play_b200/policy_epmc.py,
// which is the host statement of the same nets and the checker of this kernel (tests/test_policy_epmc.py).
//
// Training instance of the environmental level (llq_hier_policy_forward_rec): the value tower (arrays 2-46 of the shipped file), a
// Gumbel-max sample of the 256-way code head with its -log p, and the decoder on the SAMPLED code; its recurrent state per row is
// [c, h] of the code LSTM, then [c, h] of the value LSTM.
// Training instance of the strategic level (llq_hier_policy_forward_rec_strategic): the heading SAMPLED from its Gaussian head
// (mean + exp(logstd) eps, Box-Muller from Philox) with its -log p, the clipped sample feeding the frozen code controller (argmax code)
// and decoder, and the value tower of the strategic file (arrays 2-50); state per row: heading LSTM, code LSTM, value LSTM ([c, h] each).
//
// One CTA (256 threads) per 8 observation rows; activations in shared memory (89 kB), weights (1.2 MB, fp32) streamed from L2 with
// every thread of a layer reading consecutive columns and using each weight for all 8 rows; 0.23 M MAC per row on the CUDA cores.
// The recurrent states live in device memory next to the engine's arrays and are wiped where the `done` flag of the previous
// step is set.
//
// Model refresh (llq_hier_policy_set_weights, llq_hier_policy_set_pool_model): the blob is kept as given and the role tables hold
// offsets into it, so new weights of the same layout are one asynchronous copy on the caller's stream (a pool: into one model's region);
// the kernels are not involved.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/llq.h"
#include "../../include/llq_policy.h"
#include "llq_philox.cuh"

namespace {

thread_local std::string g_err_h;
int fail_h(int code, const char* msg) { g_err_h = msg; return code; }

constexpr int kThreads = 256;
constexpr int kRows = 8;                 // observation rows per CTA: every weight is read once per CTA and used for 8 rows (one warp per row
                                         // in the row-wise stages: layer norms, gates, argmax)
// roles of the weight arrays (index into the offset table the host builds from the model file)
enum Role {
  R_MEAN = 0, R_STD, R_MPROP_W, R_MPROP_B, R_MENC /* 28 arrays */, R_MEMB_W = R_MENC + 28, R_MEMB_B, R_MLSTM /* 9 */, R_LOGIT_W = R_MLSTM + 9, R_LOGIT_B,
  R_CODEBOOK, R_LLC /* 10 */, R_N_MLC = R_LLC + 10,
  R_HPROP_W = R_N_MLC, R_HPROP_B, R_HENC /* 26 */, R_HVEC = R_HENC + 26 /* 4 */, R_HEMB_W = R_HVEC + 4, R_HEMB_B, R_HLSTM /* 9 */, R_HMU_W = R_HLSTM + 9, R_HMU_B,
  R_N_ALL
};
static_assert(R_N_MLC == LLQ_HIER_ROLES_MLC && R_N_ALL == LLQ_HIER_ROLES_ALL, "role table (include/llq_policy.h)");
// the value tower's table (arrays 2-46) follows the 101 roles above in the device offset table
enum ValueRole {
  V_PROP_W = 0, V_PROP_B, V_ENC /* 28 */, V_CMD_W = V_ENC + 28, V_CMD_B, V_FC3_W, V_FC3_B, V_LSTM /* 9 */, V_OUT_W = V_LSTM + 9, V_OUT_B, V_N
};
static_assert(V_N == LLQ_HIER_ROLES_VALUE, "value-tower table (include/llq_policy.h)");
// the strategic level's training table (arrays 2-50, then the heading logstd, array 96) takes the same place
enum StrategicTrainRole {
  SV_PROP_W = 0, SV_PROP_B, SV_ENC /* 24 + fusion fc 2 */, SV_PERC_W = SV_ENC + 26, SV_PERC_B, SV_GAME /* 3 fc: 6 */, SV_CAT_W = SV_GAME + 6,
  SV_CAT_B, SV_LSTM /* 9 */, SV_OUT_W = SV_LSTM + 9, SV_OUT_B, SV_LOGSTD, SV_N
};
static_assert(SV_N == LLQ_HIER_ROLES_TRAIN_STRATEGIC, "strategic training table (include/llq_policy.h)");
constexpr int RV = R_N_ALL;
constexpr int kTrainRoles = (int)V_N > (int)SV_N ? (int)V_N : (int)SV_N;
// kernel instances: deterministic (both levels), training at the environmental level, training at the strategic level
enum Mode { M_DET = 0, M_TRAIN = 1, M_TRAIN_SEPMC = 2 };

struct Net { const float* w; const int* off; };
__device__ __forceinline__ const float* arr(const Net& n, int role) { return n.w + n.off[role]; }

// out[r][j] = act(b[j] + sum_k in[r][k] W[k][j]) for the CTA's kRows rows; W row major [K][N], N a multiple of 4, every array 16-byte
// aligned in the blob.  A thread owns FOUR consecutive columns of all rows (one 16-byte weight load and kRows shared-memory broadcasts
// per 4 x kRows FMAs); the input dimension is split into `parts` interleaved slices over the thread groups, partial sums meet in `scratch`
// (parts * kRows * N <= 4096 floats).  ACC: the sums are added to what `out` holds (b unused), so a layer too wide for one input buffer
// runs as two passes over K, the first without its activation.
template <bool ACC = false>
__device__ void dense(const float* in, int in_ld, int K, const float* W, const float* b, int N, float* out, int out_ld, float* scratch, bool relu) {
  const int t = threadIdx.x;
  const int quads = N >> 2;
  int parts = kThreads / quads; if (parts > 8) parts = 8; if (parts > 512 / N) parts = 512 / N; if (parts < 1) parts = 1;
  const int jq = t % quads, p = t / quads;
  if (p < parts) {
    float acc[kRows][4];
#pragma unroll
    for (int r = 0; r < kRows; r++) { acc[r][0] = 0.f; acc[r][1] = 0.f; acc[r][2] = 0.f; acc[r][3] = 0.f; }
    const float4* Wq = reinterpret_cast<const float4*>(W) + jq;
    int k = p;
    for (; k + 3 * parts < K; k += 4 * parts) {             // four 16-byte weight loads in flight
      float4 w[4];
#pragma unroll
      for (int u = 0; u < 4; u++) w[u] = Wq[(size_t)(k + u * parts) * quads];
#pragma unroll
      for (int u = 0; u < 4; u++) {
#pragma unroll
        for (int r = 0; r < kRows; r++) {
          const float x = in[r * in_ld + k + u * parts];
          acc[r][0] = fmaf(x, w[u].x, acc[r][0]); acc[r][1] = fmaf(x, w[u].y, acc[r][1]);
          acc[r][2] = fmaf(x, w[u].z, acc[r][2]); acc[r][3] = fmaf(x, w[u].w, acc[r][3]);
        }
      }
    }
    for (; k < K; k += parts) {
      const float4 w = Wq[(size_t)k * quads];
#pragma unroll
      for (int r = 0; r < kRows; r++) {
        const float x = in[r * in_ld + k];
        acc[r][0] = fmaf(x, w.x, acc[r][0]); acc[r][1] = fmaf(x, w.y, acc[r][1]);
        acc[r][2] = fmaf(x, w.z, acc[r][2]); acc[r][3] = fmaf(x, w.w, acc[r][3]);
      }
    }
#pragma unroll
    for (int r = 0; r < kRows; r++)
      *reinterpret_cast<float4*>(scratch + (p * kRows + r) * N + 4 * jq) = make_float4(acc[r][0], acc[r][1], acc[r][2], acc[r][3]);
  }
  __syncthreads();
  for (int idx = t; idx < kRows * N; idx += kThreads) {
    const int r = idx / N, jj = idx - r * N;
    float v = ACC ? out[r * out_ld + jj] : (b ? b[jj] : 0.f);
    for (int q = 0; q < parts; q++) v += scratch[(q * kRows + r) * N + jj];
    out[r * out_ld + jj] = relu ? fmaxf(v, 0.f) : v;
  }
  __syncthreads();
}
// TF 'SAME' convolution + ReLU on the [H][W][C] tensors of the CTA's rows in shared memory (conv1d: H = 1, kh = 1); w [kh][kw][C][O]
__device__ void conv_same_relu(const float* in, int in_ld, int H, int W, int C, const float* w, const float* b, int kh, int kw, int O, int stride,
                               float* out, int out_ld) {
  const int oh = (H + stride - 1) / stride, ow = (W + stride - 1) / stride;
  int th = (oh - 1) * stride + kh - H; if (th < 0) th = 0;
  int tw = (ow - 1) * stride + kw - W; if (tw < 0) tw = 0;
  const int pt = th / 2, pl = tw / 2, per_row = oh * ow * O;
  for (int idx = threadIdx.x; idx < kRows * per_row; idx += kThreads) {
    const int r = idx / per_row, q = idx - r * per_row;
    const int o = q % O, x = (q / O) % ow, y = q / (O * ow);
    const float* irow = in + r * in_ld;
    float acc = b[o];
    for (int di = 0; di < kh; di++) {
      const int yy = y * stride + di - pt;
      if (yy < 0 || yy >= H) continue;
      for (int dj = 0; dj < kw; dj++) {
        const int xx = x * stride + dj - pl;
        if (xx < 0 || xx >= W) continue;
        const float* ip = irow + (yy * W + xx) * C;
        const float* wp = w + ((di * kw + dj) * C) * O + o;
        for (int c = 0; c < C; c++) acc = fmaf(ip[c], wp[c * O], acc);
      }
    }
    out[r * out_ld + q] = fmaxf(acc, 0.f);
  }
  __syncthreads();
}
// first two layers of percep_2d_encoder in one pass over the raw 25 x 13 maps of all rows: 1 x 1 conv to 4 channels (+ ReLU), then 4 x 4
// stride 2 SAME (padding 1 before, 2 after; the padding belongs to the SECOND layer: padded taps contribute 0) -> [13][7][4] per row
__device__ void conv2d_first_two(const float* in, int in_ld, const float* w1, const float* b1, const float* w2, const float* b2, float* out, int out_ld) {
  for (int idx = threadIdx.x; idx < kRows * 364; idx += kThreads) {
    const int r = idx / 364, q = idx - r * 364;
    const int o = q & 3, x = (q >> 2) % 7, y = q / 28;
    const float* m = in + r * in_ld;
    float acc = b2[o];
    for (int di = 0; di < 4; di++) {
      const int yy = 2 * y + di - 1;
      if (yy < 0 || yy >= 25) continue;
      for (int dj = 0; dj < 4; dj++) {
        const int xx = 2 * x + dj - 1;
        if (xx < 0 || xx >= 13) continue;
        const float v = m[yy * 13 + xx];
        const float* wp = w2 + ((di * 4 + dj) * 4) * 4 + o;
#pragma unroll
        for (int c = 0; c < 4; c++) acc = fmaf(fmaxf(fmaf(v, w1[c], b1[c]), 0.f), wp[c * 4], acc);
      }
    }
    out[r * out_ld + q] = fmaxf(acc, 0.f);
  }
  __syncthreads();
}
// first two layers of percep_1d_encoder on the 128 lidar rays of all rows: periodic padding 4, conv1d(4 channels, k = 4, SAME), crop of the
// padded positions, conv1d(4, k = 4, stride 2, SAME: padding 1 before, 1 after) -> [64][4] per row (epmc_net.py:97-115)
__device__ void conv1d_first_two(const float* in, int in_ld, const float* w1, const float* b1, const float* w2, const float* b2, float* out, int out_ld) {
  for (int idx = threadIdx.x; idx < kRows * 256; idx += kThreads) {
    const int r = idx >> 8, q = idx & 255;
    const int o = q & 3, x = q >> 2;
    const float* ray = in + r * in_ld;
    float acc = b2[o];
    for (int dj = 0; dj < 4; dj++) {
      const int ii = 2 * x + dj - 1;                        // position in the cropped first-layer output
      if (ii < 0 || ii >= 128) continue;
      // first layer at padded position ii + 4: taps at padded positions ii + 3 .. ii + 6, i.e. rays (ii - 1 .. ii + 2) mod 128
      const float p0 = ray[(ii + 127) & 127], p1 = ray[ii], p2 = ray[(ii + 1) & 127], p3 = ray[(ii + 2) & 127];
#pragma unroll
      for (int c = 0; c < 4; c++) {
        const float a = fmaxf(fmaf(p0, w1[c], fmaf(p1, w1[4 + c], fmaf(p2, w1[8 + c], fmaf(p3, w1[12 + c], b1[c])))), 0.f);
        acc = fmaf(a, w2[(dj * 4 + c) * 4 + o], acc);
      }
    }
    out[r * out_ld + q] = fmaxf(acc, 0.f);
  }
  __syncthreads();
}
// the three perception encoders of one usr_cmd_encoder for every row of the CTA: enc[0..8) 2-D map, [8..16) lidar, [16..24) front map;
// row r's 88 features go to cat + r * cat_ld.  bufa [kRows][364], bufb [kRows][128].
__device__ void perception(const Net& n, int enc, const float* obs, int obs_ld, float* bufa, float* bufb, float* cat, int cat_ld) {
  for (int map = 0; map < 2; map++) {
    const int e = enc + (map == 0 ? 0 : 16);
    conv2d_first_two(obs + (map == 0 ? 135 : 588), obs_ld, arr(n, e), arr(n, e + 1), arr(n, e + 2), arr(n, e + 3), bufa, 364);      // 13 x 7 x 4
    conv_same_relu(bufa, 364, 13, 7, 4, arr(n, e + 4), arr(n, e + 5), 2, 2, 4, 2, bufb, 128);                                       // 7 x 4 x 4
    conv_same_relu(bufb, 128, 7, 4, 4, arr(n, e + 6), arr(n, e + 7), 2, 2, 1, 1, cat + (map == 0 ? 0 : 60), cat_ld);                // 28
  }
  const int e = enc + 8;
  conv1d_first_two(obs + 460, obs_ld, arr(n, e), arr(n, e + 1), arr(n, e + 2), arr(n, e + 3), bufa, 364);                           // 64 x 4
  conv_same_relu(bufa, 364, 1, 64, 4, arr(n, e + 4), arr(n, e + 5), 1, 4, 4, 2, bufb, 128);                                         // 32 x 4
  conv_same_relu(bufb, 128, 1, 32, 4, arr(n, e + 6), arr(n, e + 7), 1, 4, 1, 1, cat + 28, cat_ld);                                  // 32
}
// layer norm over n values of every row (warp r normalises row r): v <- (v - mean) / sqrt(var + 1e-12) * g + b (tf.contrib.layers.layer_norm)
__device__ void layer_norm(float* v, int ld, int n, const float* beta, const float* gamma) {
  const int r = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (r < kRows) {
    float* x = v + r * ld;
    float s = 0.f;
    for (int i = l; i < n; i += 32) s += x[i];
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float m = s / (float)n;
    float q = 0.f;
    for (int i = l; i < n; i += 32) { const float d = x[i] - m; q = fmaf(d, d, q); }
    for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float inv = 1.0f / sqrtf(q / (float)n + 1e-12f);
    for (int i = l; i < n; i += 32) x[i] = (x[i] - m) * inv * gamma[i] + beta[i];
  }
  __syncthreads();
}
// one step of the layer-norm LSTM (nh = 32) for every row: x [kRows][256] in shared memory, state [c(32), h(32)] per row in global memory
// (updated in place; rows with live[r] == 0 are not stored; row r's state is state + rows.srow(r) * state_ld, see BlockRows); arrays
// lstm + 0..8 = wx, wh, b, beta_x, gamma_x, beta_h, gamma_h, beta_c, gamma_c.  Leaves h in hout[kRows][32].
template <class Rows>
__device__ void lstm_step(const Net& n, int lstm, const float* x, float* state, int state_ld, const Rows& rows, const int* live, const int* wipe,
                          float* zx, float* zh, float* cbuf, float* hout, float* scratch) {
  const int t = threadIdx.x;
  for (int idx = t; idx < kRows * 64; idx += kThreads) {
    const int r = idx >> 6, i = idx & 63;
    cbuf[idx] = (live[r] && !wipe[r]) ? state[(size_t)rows.srow(r) * state_ld + i] : 0.f;          // cbuf[r][0..32) = c, [32..64) = h
  }
  __syncthreads();
  dense(x, 256, 256, arr(n, lstm), nullptr, 128, zx, 128, scratch, false);
  dense(cbuf + 32, 64, 32, arr(n, lstm + 1), nullptr, 128, zh, 128, scratch, false);
  layer_norm(zx, 128, 128, arr(n, lstm + 3), arr(n, lstm + 4));
  layer_norm(zh, 128, 128, arr(n, lstm + 5), arr(n, lstm + 6));
  const int r = t >> 5, u = t & 31;                         // 8 rows x 32 units
  {
    const float* b = arr(n, lstm + 2);
    float* px = zx + r * 128; float* ph = zh + r * 128;
    const float gi = px[u] + ph[u] + b[u], gf = px[32 + u] + ph[32 + u] + b[32 + u];
    const float go = px[64 + u] + ph[64 + u] + b[64 + u], gu = px[96 + u] + ph[96 + u] + b[96 + u];
    const float c = (1.0f / (1.0f + expf(-(gf + 1.0f)))) * cbuf[r * 64 + u] + (1.0f / (1.0f + expf(-gi))) * tanhf(gu);      // forget_bias 1
    __syncwarp();
    cbuf[r * 64 + u] = c;
    px[u] = c;                                               // layer norm of the new cell state (32 values)
    ph[u] = 1.0f / (1.0f + expf(-go));
    if (live[r]) state[(size_t)rows.srow(r) * state_ld + u] = c;
  }
  __syncthreads();
  layer_norm(zx, 128, 32, arr(n, lstm + 7), arr(n, lstm + 8));
  {
    const float h = zh[r * 128 + u] * tanhf(zx[r * 128 + u]);
    hout[r * 32 + u] = h;
    if (live[r]) state[(size_t)rows.srow(r) * state_ld + 32 + u] = h;
  }
  __syncthreads();
}

constexpr int kObsLd = 968;      // shared-memory row stride of the observation block
struct alignas(16) Smem {
  float scr[4096];                 // partial sums of the split layers (parts * rows * N <= 4096); first member: 16-byte aligned
  float obs[kRows][kObsLd];
  float p[kRows][136];
  float cat[kRows][256], x[kRows][256], y[kRows][256];
  float zx[kRows][128], zh[kRows][128], c[kRows][64], h[kRows][32];
  float a[kRows * 364], b[kRows * 128];   // convolution buffers: [13][7][4] / [64][4] and [7][4][4] / [32][4] per row
  float ang[kRows];
  int code[kRows], live[kRows], wipe[kRows];
};

// outputs and noise key of the training instance (unused by the deterministic one)
struct Sample { float* values; float* neglogp; long long out_ld; unsigned long long seed, counter; long long row_gid0; };

// g = -log(-log u) of one Philox word: u = (r + 1/2) 2^-32 in fp32, clamped below 1 (r >= 2^32 - 128 rounds to 1.0f, g would be +inf)
__device__ __forceinline__ float gumbel(uint32_t r) {
  const float u = fminf(((float)r + 0.5f) * 2.3283064365386963e-10f, 0.99999994f);
  return -logf(-logf(u));
}

// Box-Muller pair of two Philox words with the conversions of llq_policy.cu's Gaussian action noise: u0 = (ra + 1/2) 2^-32 in fp32,
// clamped below 1 (ra >= 2^32 - 128 rounds to 1.0f), u1 = rb 2^-32; returns sqrt(-2 log u0) (cos, sin)(2 pi u1).  (llq_policy.cu keeps
// its inline form: calling this there changes that kernel's instruction schedule.)
__device__ __forceinline__ float2 box_muller(uint32_t ra, uint32_t rb) {
  const float u0 = ((float)ra + 0.5f) * 2.3283064365386963e-10f, u1 = (float)rb * 2.3283064365386963e-10f;
  const float rad = sqrtf(-2.0f * logf(fminf(u0, 0.99999994f)));
  float s, c;
  sincosf(6.283185307179586f * u1, &s, &c);
  return make_float2(rad * c, rad * s);
}

// the 29 game-vector slots of every row (percept_vec | oppo_info | flag_info | with_flag) -> x[r][0..29)
__device__ __forceinline__ void game_vector(Smem& S) {
  for (int idx = threadIdx.x; idx < kRows * 29; idx += kThreads) {
    const int r = idx / 29, i = idx - r * 29;
    S.x[r][i] = i < 5 ? S.obs[r][913 + i] : (i < 20 ? S.obs[r][918 + i - 5] : (i < 27 ? S.obs[r][948 + i - 20] : S.obs[r][962 + i - 27]));
  }
  __syncthreads();
}

// The rows of a CTA.  BlockRows: rows row0 .. row0 + 7 of the batch (hier_policy_kernel).  ListRows: the entries of a pool segment
// (hier_pool_kernel), row ids in shared memory, -1 for a pad entry.  row(r) indexes the batch (observation, done, outputs); the state of
// row r is at state + (base() + srow(r)) * ssz.
struct BlockRows {
  int row0, n;
  __device__ __forceinline__ bool live(int r) const { return row0 + r < n; }
  __device__ __forceinline__ int row(int r) const { return row0 + r; }
  __device__ __forceinline__ int srow(int r) const { return r; }
  __device__ __forceinline__ int base() const { return row0; }
};
struct ListRows {
  const int* id;
  __device__ __forceinline__ bool live(int r) const { return id[r] >= 0; }
  __device__ __forceinline__ int row(int r) const { return id[r]; }
  __device__ __forceinline__ int srow(int r) const { return id[r]; }
  __device__ __forceinline__ int base() const { return 0; }
};

// The policy forward of one CTA's rows.  The training modes run on BlockRows only (their noise is keyed by rows.row0).
template <int MODE, class Rows>
__device__ __forceinline__ void policy_rows(Smem& S, const Rows& rows, Net net, int strategic, const float* __restrict__ obs, long long obs_ld,
                                            const unsigned char* __restrict__ done, float* __restrict__ state, float* __restrict__ actions,
                                            int* __restrict__ codes, float* __restrict__ heading, const Sample& smp) {
  const int t = threadIdx.x;
  if constexpr (MODE == M_TRAIN) strategic = 0;
  if constexpr (MODE == M_TRAIN_SEPMC) strategic = 1;
  const int ow = strategic ? 965 : 916;
  if (t < kRows) {
    const int live = rows.live(t);
    S.live[t] = live;
    S.wipe[t] = live && done != nullptr && done[rows.row(t)] != 0;
  }
  for (int idx = t; idx < kRows * kObsLd; idx += kThreads) {
    const int r = idx / kObsLd, i = idx - r * kObsLd;
    S.obs[r][i] = (rows.live(r) && i < ow) ? obs[(size_t)rows.row(r) * obs_ld + i] : 0.f;
  }
  __syncthreads();
  for (int idx = t; idx < kRows * 135; idx += kThreads) {
    const int r = idx / 135, i = idx - r * 135;
    S.p[r][i] = fminf(fmaxf((S.obs[r][i] - arr(net, R_MEAN)[i]) / (arr(net, R_STD)[i] + 1e-8f), -5.f), 5.f);
  }
  __syncthreads();
  const int ssz = MODE == M_TRAIN_SEPMC ? 192 : ((MODE == M_TRAIN || strategic) ? 128 : 64);
  float* st = state + (size_t)rows.base() * ssz;
  if (strategic) {
    // ---- heading controller
    dense(&S.p[0][0], 136, 135, arr(net, R_HPROP_W), arr(net, R_HPROP_B), 64, &S.cat[0][0], 256, S.scr, true);              // cat[0..64)
    perception(net, R_HENC, &S.obs[0][0], kObsLd, S.a, S.b, &S.x[0][0], 256);                                                // x[0..88)
    dense(&S.x[0][0], 256, 88, arr(net, R_HENC + 24), arr(net, R_HENC + 25), 64, &S.cat[0][64], 256, S.scr, true);          // cat[64..128)
    game_vector(S);
    dense(&S.x[0][0], 256, 29, arr(net, R_HVEC), arr(net, R_HVEC + 1), 64, &S.y[0][0], 256, S.scr, true);
    dense(&S.y[0][0], 256, 64, arr(net, R_HVEC + 2), arr(net, R_HVEC + 3), 64, &S.cat[0][128], 256, S.scr, true);           // cat[128..192)
    dense(&S.cat[0][0], 256, 192, arr(net, R_HEMB_W), arr(net, R_HEMB_B), 256, &S.x[0][0], 256, S.scr, true);
    lstm_step(net, R_HLSTM, &S.x[0][0], st, ssz, rows, S.live, S.wipe, &S.zx[0][0], &S.zh[0][0], &S.c[0][0], &S.h[0][0], S.scr);
    if (t < kRows) {
      float a = arr(net, R_HMU_B)[0];
      for (int k = 0; k < 32; k++) a = fmaf(S.h[t][k], arr(net, R_HMU_W)[k], a);
      if constexpr (MODE == M_TRAIN_SEPMC) {
        // heading sample a = mu + exp(logstd) eps: eps from Philox keyed (global row, q = 64, counter) / seed (q 0..63 are the Gumbel draws'
        // of the environmental level); the record gets the raw a and -log p of the raw a, the code controller the clipped one
        const uint4 r = philox4x32(make_uint4((uint32_t)(smp.row_gid0 + rows.row0 + t), 64u, (uint32_t)smp.counter, (uint32_t)(smp.counter >> 32)),
                                   make_uint2((uint32_t)smp.seed, (uint32_t)(smp.seed >> 32)));
        const float eps = box_muller(r.x, r.y).x, ls = arr(net, RV + SV_LOGSTD)[0];
        a = fmaf(expf(ls), eps, a);
        if (S.live[t]) {
          if (heading) heading[(size_t)(rows.row0 + t) * smp.out_ld] = a;
          if (smp.neglogp) smp.neglogp[(size_t)(rows.row0 + t) * smp.out_ld] = 0.5f * eps * eps + ls + 0.91893853320467274f;   // + 0.5 log(2 pi)
        }
        S.ang[t] = fminf(fmaxf(a, -3.14159265358979f), 3.14159265358979f);
      } else {
        a = fminf(fmaxf(a, -3.14159265358979f), 3.14159265358979f);
        S.ang[t] = a;
        if (heading && S.live[t]) heading[rows.row(t)] = a;
      }
    }
    __syncthreads();
    st += 64;
  }
  if constexpr (MODE == M_TRAIN) {
    // ---- value tower (arrays 2-46), wired like the code controller: [prop 135 -> 128 | command encoder -> 64 -> 128] -> 256 -> LSTM(32)
    // -> V (linear); its [c, h] is the second half of the row's state
    dense(&S.p[0][0], 136, 135, arr(net, RV + V_PROP_W), arr(net, RV + V_PROP_B), 128, &S.cat[0][0], 256, S.scr, true);       // cat[0..128)
    if (t < kRows * 3) {
      const int r = t / 3, i = t - 3 * r;
      S.y[r][i] = S.obs[r][913 + i];
    }
    __syncthreads();
    dense(&S.y[0][0], 256, 3, arr(net, RV + V_ENC + 24), arr(net, RV + V_ENC + 25), 32, &S.x[0][0], 256, S.scr, true);       // x[0..32)
    perception(net, RV + V_ENC, &S.obs[0][0], kObsLd, S.a, S.b, &S.x[0][32], 256);                                          // x[32..120)
    dense(&S.x[0][0], 256, 120, arr(net, RV + V_ENC + 26), arr(net, RV + V_ENC + 27), 64, &S.y[0][0], 256, S.scr, true);     // y[0..64)
    dense(&S.y[0][0], 256, 64, arr(net, RV + V_CMD_W), arr(net, RV + V_CMD_B), 128, &S.cat[0][128], 256, S.scr, true);       // cat[128..256)
    dense(&S.cat[0][0], 256, 256, arr(net, RV + V_FC3_W), arr(net, RV + V_FC3_B), 256, &S.x[0][0], 256, S.scr, true);
    lstm_step(net, RV + V_LSTM, &S.x[0][0], st + 64, ssz, rows, S.live, S.wipe, &S.zx[0][0], &S.zh[0][0], &S.c[0][0], &S.h[0][0], S.scr);
    if (t < kRows) {
      float v = arr(net, RV + V_OUT_B)[0];
      for (int k = 0; k < 32; k++) v = fmaf(S.h[t][k], arr(net, RV + V_OUT_W)[k], v);
      if (smp.values && S.live[t]) smp.values[(size_t)(rows.row0 + t) * smp.out_ld] = v;
    }
    __syncthreads();
  }
  if constexpr (MODE == M_TRAIN_SEPMC) {
    // ---- value tower of the strategic level (arrays 2-50), in the heading controller's [prop | perception | game] order: prop 135 -> 128 |
    // perception encoder 88 -> 64 -> 128 | game vector 29 -> 64 -> 64 -> 128, concatenated 384 -> 256 (two passes over K: cat holds 256)
    // -> LSTM(32) -> V (linear); its [c, h] is the third part of the row's state
    dense(&S.p[0][0], 136, 135, arr(net, RV + SV_PROP_W), arr(net, RV + SV_PROP_B), 128, &S.cat[0][0], 256, S.scr, true);     // cat[0..128)
    perception(net, RV + SV_ENC, &S.obs[0][0], kObsLd, S.a, S.b, &S.x[0][0], 256);                                          // x[0..88)
    dense(&S.x[0][0], 256, 88, arr(net, RV + SV_ENC + 24), arr(net, RV + SV_ENC + 25), 64, &S.y[0][0], 256, S.scr, true);    // y[0..64)
    dense(&S.y[0][0], 256, 64, arr(net, RV + SV_PERC_W), arr(net, RV + SV_PERC_B), 128, &S.cat[0][128], 256, S.scr, true);   // cat[128..256)
    game_vector(S);                                                                                                        // x[0..29)
    dense(&S.x[0][0], 256, 29, arr(net, RV + SV_GAME), arr(net, RV + SV_GAME + 1), 64, &S.y[0][0], 256, S.scr, true);
    dense(&S.y[0][0], 256, 64, arr(net, RV + SV_GAME + 2), arr(net, RV + SV_GAME + 3), 64, &S.x[0][0], 256, S.scr, true);
    dense(&S.x[0][0], 256, 64, arr(net, RV + SV_GAME + 4), arr(net, RV + SV_GAME + 5), 128, &S.y[0][0], 256, S.scr, true);   // y[0..128)
    dense(&S.cat[0][0], 256, 256, arr(net, RV + SV_CAT_W), arr(net, RV + SV_CAT_B), 256, &S.x[0][0], 256, S.scr, false);     // rows 0-255
    dense<true>(&S.y[0][0], 256, 128, arr(net, RV + SV_CAT_W) + 256 * 256, nullptr, 256, &S.x[0][0], 256, S.scr, true);    // rows 256-383
    lstm_step(net, RV + SV_LSTM, &S.x[0][0], st + 64, ssz, rows, S.live, S.wipe, &S.zx[0][0], &S.zh[0][0], &S.c[0][0], &S.h[0][0], S.scr);
    if (t < kRows) {
      float v = arr(net, RV + SV_OUT_B)[0];
      for (int k = 0; k < 32; k++) v = fmaf(S.h[t][k], arr(net, RV + SV_OUT_W)[k], v);
      if (smp.values && S.live[t]) smp.values[(size_t)(rows.row0 + t) * smp.out_ld] = v;
    }
    __syncthreads();
  }
  // ---- code controller (environmental level)
  dense(&S.p[0][0], 136, 135, arr(net, R_MPROP_W), arr(net, R_MPROP_B), 64, &S.cat[0][0], 256, S.scr, true);                // cat[0..64)
  if (t < kRows * 3) {
    const int r = t / 3, i = t - 3 * r;
    S.y[r][i] = strategic ? (i == 0 ? cosf(S.ang[r]) : (i == 1 ? sinf(S.ang[r]) : S.obs[r][964])) : S.obs[r][913 + i];
  }
  __syncthreads();
  dense(&S.y[0][0], 256, 3, arr(net, R_MENC + 24), arr(net, R_MENC + 25), 32, &S.x[0][0], 256, S.scr, true);                // x[0..32) = target embedding
  perception(net, R_MENC, &S.obs[0][0], kObsLd, S.a, S.b, &S.x[0][32], 256);                                                // x[32..120)
  dense(&S.x[0][0], 256, 120, arr(net, R_MENC + 26), arr(net, R_MENC + 27), 64, &S.cat[0][64], 256, S.scr, true);           // cat[64..128)
  dense(&S.cat[0][0], 256, 128, arr(net, R_MEMB_W), arr(net, R_MEMB_B), 256, &S.x[0][0], 256, S.scr, true);
  lstm_step(net, R_MLSTM, &S.x[0][0], st, ssz, rows, S.live, S.wipe, &S.zx[0][0], &S.zh[0][0], &S.c[0][0], &S.h[0][0], S.scr);
  dense(&S.h[0][0], 32, 32, arr(net, R_LOGIT_W), arr(net, R_LOGIT_B), 256, &S.y[0][0], 256, S.scr, false);                  // logits
  if constexpr (MODE == M_TRAIN) {
    // Gumbel-max sample: code = argmax_j (logit_j + g_j), g from Philox keyed (global row, q, counter) / seed, one call per four logits
    for (int idx = t; idx < kRows * 64; idx += kThreads) {
      const int r = idx >> 6, q = idx & 63;
      const uint4 b = philox4x32(make_uint4((uint32_t)(smp.row_gid0 + rows.row0 + r), (uint32_t)q, (uint32_t)smp.counter, (uint32_t)(smp.counter >> 32)),
                                 make_uint2((uint32_t)smp.seed, (uint32_t)(smp.seed >> 32)));
      *reinterpret_cast<float4*>(&S.x[r][4 * q]) = make_float4(gumbel(b.x), gumbel(b.y), gumbel(b.z), gumbel(b.w));
    }
    __syncthreads();
    const int r = t >> 5, l = t & 31;
    float best = -3.4e38f, m = -3.4e38f; int bi = 0;
    for (int i = l; i < 256; i += 32) {
      const float v = S.y[r][i] + S.x[r][i];
      if (v > best) { best = v; bi = i; }
      m = fmaxf(m, S.y[r][i]);
    }
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
      m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    }
    float se = 0.f;                                         // -log p = (m - l_code) + log sum exp(l_j - m): no overflow for large logits
    for (int i = l; i < 256; i += 32) se += expf(S.y[r][i] - m);
    for (int o = 16; o > 0; o >>= 1) se += __shfl_xor_sync(0xffffffffu, se, o);
    if (l == 0) {
      S.code[r] = bi;
      if (S.live[r]) {
        if (codes) codes[rows.row0 + r] = bi;
        if (smp.neglogp) smp.neglogp[(size_t)(rows.row0 + r) * smp.out_ld] = (m - S.y[r][bi]) + logf(se);
      }
    }
  } else {                                                  // argmax per row (warp r), first occurrence
    const int r = t >> 5, l = t & 31;
    float best = -3.4e38f; int bi = 0;
    for (int i = l; i < 256; i += 32) if (S.y[r][i] > best) { best = S.y[r][i]; bi = i; }
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    if (l == 0) { S.code[r] = bi; if (codes && S.live[r]) codes[rows.row(r)] = bi; }
  }
  __syncthreads();
  // ---- frozen primitive-level decoder
  { const int r = t >> 5, u = t & 31; S.y[r][u] = arr(net, R_CODEBOOK)[u * 256 + S.code[r]]; }
  __syncthreads();
  dense(&S.p[0][0], 136, 135, arr(net, R_LLC), arr(net, R_LLC + 1), 64, &S.cat[0][0], 256, S.scr, true);
  dense(&S.y[0][0], 256, 32, arr(net, R_LLC + 2), arr(net, R_LLC + 3), 32, &S.cat[0][64], 256, S.scr, true);
  dense(&S.cat[0][0], 256, 96, arr(net, R_LLC + 4), arr(net, R_LLC + 5), 256, &S.x[0][0], 256, S.scr, true);
  dense(&S.x[0][0], 256, 256, arr(net, R_LLC + 6), arr(net, R_LLC + 7), 256, &S.y[0][0], 256, S.scr, true);
  dense(&S.y[0][0], 256, 256, arr(net, R_LLC + 8), arr(net, R_LLC + 9), 12, &S.x[0][0], 256, S.scr, false);
  if (t < kRows * 12) {
    const int r = t / 12, i = t - 12 * r;
    if (S.live[r]) actions[(size_t)rows.row(r) * 12 + i] = S.x[r][i];
  }
}

template <int MODE>
__global__ void __launch_bounds__(kThreads) hier_policy_kernel(Net net, int strategic, const float* __restrict__ obs, long long obs_ld, int n_rows,
                                                               const unsigned char* __restrict__ done, float* __restrict__ state, float* __restrict__ actions,
                                                               int* __restrict__ codes, float* __restrict__ heading, Sample smp) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  policy_rows<MODE>(*reinterpret_cast<Smem*>(smem_raw), BlockRows{(int)blockIdx.x * kRows, n_rows}, net, strategic, obs, obs_ld, done, state, actions,
                    codes, heading, smp);
}

// ---- opponent pool (llq_hier_policy_forward_pool): K deterministic strategic-level models, every row run with its own model
constexpr int kAssignThreads = 1024;
// model k is drawn for r < t[k] (and r >= t[k - 1]); t[K - 1] = 2^32; by value, so a new table takes effect at the next launch
struct Cutoffs { unsigned long long t[LLQ_HIER_POOL_MAX]; };
// the pool kernel's shared memory: Smem, then the row ids of the CTA's segment entries
struct PoolSmem : Smem { int rid[kRows]; };

// One CTA.  Draws a model for every row with done[i] != 0 (r = word x of Philox4x32-10, counter (low 32 bits of row_gid0 + i, 65,
// counter lo, counter hi), key (seed lo, seed hi); model = the smallest k with r < t[k]), records every row's model (-1 outside
// [0, K)), and buckets the rows by model: segment k holds its rows in ascending order, padded with -1 to a multiple of kRows, and
// starts at CTA seg_cta[k] of the pool forward (seg_cta[K] = the CTAs of all segments); its entries are seg_rows[seg_cta[k] * kRows ..).
__global__ void __launch_bounds__(kAssignThreads) hier_pool_assign_kernel(int n, int n_models, Cutoffs cut, const unsigned char* __restrict__ done,
                                                                          int* __restrict__ model, float* __restrict__ rec, long long rec_ld,
                                                                          unsigned long long seed, unsigned long long counter, long long row_gid0,
                                                                          int* __restrict__ seg_cta, int* __restrict__ seg_rows) {
  __shared__ int cnt[LLQ_HIER_POOL_MAX], first[LLQ_HIER_POOL_MAX], fill[LLQ_HIER_POOL_MAX];
  __shared__ int chunk[kAssignThreads];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  if (t < LLQ_HIER_POOL_MAX) { cnt[t] = 0; fill[t] = 0; }
  __syncthreads();
  for (int i = t; i < n; i += kAssignThreads) {
    int m = model[i];
    if (done != nullptr && done[i] != 0) {
      const uint32_t r = philox4x32(make_uint4((uint32_t)(row_gid0 + i), 65u, (uint32_t)counter, (uint32_t)(counter >> 32)),
                                    make_uint2((uint32_t)seed, (uint32_t)(seed >> 32))).x;
      m = 0;                                                 // the cutoffs do not decrease: the count of t[k] <= r is the smallest k with r < t[k]
#pragma unroll
      for (int k = 0; k < LLQ_HIER_POOL_MAX - 1; k++) m += (k < n_models - 1 && (unsigned long long)r >= cut.t[k]) ? 1 : 0;
      model[i] = m;
    }
    const bool in = m >= 0 && m < n_models;
    if (rec != nullptr) rec[(size_t)i * rec_ld] = in ? (float)m : -1.f;
    if (in) atomicAdd(&cnt[m], 1);
  }
  __syncthreads();
  if (t == 0) {
    int c = 0;
    for (int k = 0; k < n_models; k++) { first[k] = c; seg_cta[k] = c; c += (cnt[k] + kRows - 1) / kRows; }
    seg_cta[n_models] = c;
  }
  __syncthreads();
  // stable placement, kAssignThreads rows at a time: warp w places the rows of models w, w + 32 in ascending order (a ballot per 32 rows)
  for (int c0 = 0; c0 < n; c0 += kAssignThreads) {
    const int len = min(kAssignThreads, n - c0);
    chunk[t] = t < len ? model[c0 + t] : -1;                 // thread t wrote model[c0 + t] above: its own write
    __syncthreads();
    for (int k = warp; k < n_models; k += kAssignThreads / 32) {
      int pos = fill[k];
      for (int s = 0; s < len; s += 32) {
        const bool mine = chunk[s + lane] == k;
        const unsigned bal = __ballot_sync(0xffffffffu, mine);
        if (mine) seg_rows[first[k] * kRows + pos + __popc(bal & ((1u << lane) - 1u))] = c0 + s + lane;
        pos += __popc(bal);
      }
      if (lane == 0) fill[k] = pos;
    }
    __syncthreads();
  }
  if (t < n_models)
    for (int j = cnt[t]; j % kRows; j++) seg_rows[first[t] * kRows + j] = -1;
}

// The deterministic strategic-level forward of a pool: CTA b runs the kRows entries seg_rows[b * kRows ..) of its segment k (the largest
// k with seg_cta[k] <= b) with model k, whose offset table is off + k * RV; CTAs from seg_cta[K] on return at once.
__global__ void __launch_bounds__(kThreads) hier_pool_kernel(const float* __restrict__ w, const int* __restrict__ off, int n_models,
                                                             const int* __restrict__ seg_cta, const int* __restrict__ seg_rows,
                                                             const float* __restrict__ obs, long long obs_ld, const unsigned char* __restrict__ done,
                                                             float* __restrict__ state, float* __restrict__ actions, int* __restrict__ codes,
                                                             float* __restrict__ heading) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  PoolSmem& S = *reinterpret_cast<PoolSmem*>(smem_raw);
  const int b = blockIdx.x;
  if (b >= seg_cta[n_models]) return;
  int k = 0;
  for (int j = 1; j < n_models; j++) if (seg_cta[j] <= b) k = j;
  if (threadIdx.x < kRows) S.rid[threadIdx.x] = seg_rows[b * kRows + threadIdx.x];
  __syncthreads();
  policy_rows<M_DET>(S, ListRows{S.rid}, Net{w, off + k * RV}, 1, obs, obs_ld, done, state, actions, codes, heading, Sample{});
}

}  // namespace

struct llq_hier_policy {
  int device = 0, strategic = 0, train = 0;
  bool attr_set = false;
  float* d_w = nullptr;
  int64_t n_weights = 0;                                     // the blob's length, fixed at create
  int* d_off = nullptr;
  // pool handles (llq_hier_policy_create_pool): K models, the cutoffs of the next draws, the assign kernel's workspace
  int n_models = 0, max_rows = 0;
  Cutoffs cut{};
  int* d_seg = nullptr;                                      // [K + 1] first CTA of every segment, then the segments' row ids
  // model k of a pool owns the blob floats [region[k], region_end[k]) (pool_regions); regions_ok = false: two models share arrays
  std::vector<int64_t> region, region_end;
  bool regions_ok = false;
  // host refreshes: pinned staging (stage_len floats), its upload followed by ev_stage
  float* h_stage = nullptr;
  int64_t stage_len = 0;
  cudaEvent_t ev_stage = nullptr;
  bool staged = false;
};

namespace {

// the device checks and the upload of the blob and of the device offset table `off`, once the arguments are checked
int upload(const float* weights, int64_t n_weights, const std::vector<int>& off, int32_t strategic, int train, int32_t device,
           llq_hier_policy_handle* out) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail_h(LLQ_ECUDA, "no CUDA device visible (no CPU fallback)");
  if (device < 0 || device >= ndev) return fail_h(LLQ_EINVAL, "device ordinal out of range");
  if (cudaSetDevice(device) != cudaSuccess) return fail_h(LLQ_ECUDA, "cudaSetDevice failed");
  llq_hier_policy* h = new (std::nothrow) llq_hier_policy();
  if (!h) return fail_h(LLQ_ENOMEM, "out of memory");
  h->device = device; h->strategic = strategic ? 1 : 0; h->train = train; h->n_weights = n_weights;
  if (cudaMalloc(&h->d_w, sizeof(float) * (size_t)n_weights) != cudaSuccess || cudaMalloc(&h->d_off, sizeof(int) * off.size()) != cudaSuccess ||
      cudaMemcpy(h->d_w, weights, sizeof(float) * (size_t)n_weights, cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy(h->d_off, off.data(), sizeof(int) * off.size(), cudaMemcpyHostToDevice) != cudaSuccess) {
    cudaFree(h->d_w); cudaFree(h->d_off); delete h;
    return fail_h(LLQ_ECUDA, "weight upload failed");
  }
  *out = h;
  return LLQ_OK;
}

// `value_offsets` (n_value entries: LLQ_HIER_ROLES_VALUE, or LLQ_HIER_ROLES_TRAIN_STRATEGIC at the strategic level) null: a deterministic
// handle
int create(const float* weights, int64_t n_weights, const int32_t* offsets, int32_t n_roles, const int32_t* value_offsets, int32_t n_value,
           int32_t strategic, int32_t device, llq_hier_policy_handle* out) {
  if (!weights || !offsets || !out) return fail_h(LLQ_EINVAL, "null argument");
  if (n_roles != (strategic ? LLQ_HIER_ROLES_ALL : LLQ_HIER_ROLES_MLC)) return fail_h(LLQ_EINVAL, "role table has the wrong length (include/llq_policy.h)");
  for (int i = 0; i < n_roles; i++) if (offsets[i] < 0 || offsets[i] >= n_weights) return fail_h(LLQ_EINVAL, "role offset outside the weight blob");
  if (value_offsets)
    for (int i = 0; i < n_value; i++)
      if (value_offsets[i] < 0 || value_offsets[i] >= n_weights) return fail_h(LLQ_EINVAL, "training-table offset outside the weight blob");
  std::vector<int> off(RV + kTrainRoles, 0);
  for (int i = 0; i < n_roles; i++) off[i] = offsets[i];
  if (value_offsets) for (int i = 0; i < n_value; i++) off[RV + i] = value_offsets[i];
  return upload(weights, n_weights, off, strategic, value_offsets ? 1 : 0, device, out);
}

// the cutoffs of probs[0..K) (checked by the caller): sequential fp64 sums, t_k = floor(cum_k / cum_{K-1} 2^32), t_{K-1} = 2^32
Cutoffs cutoffs(const double* probs, int K) {
  Cutoffs c{};
  double cum[LLQ_HIER_POOL_MAX], s = 0.0;
  for (int k = 0; k < K; k++) { s += probs[k]; cum[k] = s; }
  for (int k = 0; k < K - 1; k++) c.t[k] = (unsigned long long)std::floor(cum[k] / s * 4294967296.0);
  c.t[K - 1] = 1ull << 32;
  return c;
}

// model k's region of a pool blob: from its smallest role offset to the next larger model start (or the blob's end); false when two models
// start at the same float or one of model k's arrays starts outside its region (two models sharing arrays)
bool pool_regions(const int32_t* offsets, int K, int64_t n_weights, std::vector<int64_t>& lo, std::vector<int64_t>& hi) {
  lo.assign(K, 0); hi.assign(K, n_weights);
  for (int k = 0; k < K; k++) {
    lo[k] = offsets[(size_t)k * RV];
    for (int r = 1; r < RV; r++) lo[k] = std::min<int64_t>(lo[k], offsets[(size_t)k * RV + r]);
  }
  for (int k = 0; k < K; k++)
    for (int j = 0; j < K; j++) {
      if (j != k && lo[j] == lo[k]) return false;
      if (lo[j] > lo[k]) hi[k] = std::min(hi[k], lo[j]);
    }
  for (int k = 0; k < K; k++)
    for (int r = 0; r < RV; r++)
      if (offsets[(size_t)k * RV + r] >= hi[k]) return false;
  return true;
}

// copies n floats of `weights` (host: through the handle's pinned staging; device: checked to lie on the handle's device) to the blob at
// float `dst`, on `stream`
int refresh(llq_hier_policy_handle h, int64_t dst, const float* weights, int64_t n, int32_t on_device, void* stream) {
  if (on_device != 0 && on_device != 1) return fail_h(LLQ_EINVAL, "on_device must be 0 (host memory) or 1 (device memory)");
  if (cudaSetDevice(h->device) != cudaSuccess) return fail_h(LLQ_ECUDA, "cudaSetDevice failed");
  const cudaStream_t s = (cudaStream_t)stream;
  const size_t bytes = sizeof(float) * (size_t)n;
  if (on_device) {
    cudaPointerAttributes a{};
    if (cudaPointerGetAttributes(&a, weights) != cudaSuccess || a.type != cudaMemoryTypeDevice || a.device != h->device) {
      cudaGetLastError();
      return fail_h(LLQ_EINVAL, "on_device = 1 needs device memory on the handle's device");
    }
    if (cudaMemcpyAsync(h->d_w + dst, weights, bytes, cudaMemcpyDeviceToDevice, s) != cudaSuccess) return fail_h(LLQ_ECUDA, "weight copy failed");
    return LLQ_OK;
  }
  if (h->stage_len < n) {                                    // the first host refresh (a pool's regions may differ in length)
    if (h->staged && cudaEventSynchronize(h->ev_stage) != cudaSuccess) return fail_h(LLQ_ECUDA, "staging event failed");
    if (h->h_stage) cudaFreeHost(h->h_stage);
    h->h_stage = nullptr; h->stage_len = 0; h->staged = false;
    if (cudaHostAlloc(&h->h_stage, bytes, cudaHostAllocDefault) != cudaSuccess) return fail_h(LLQ_ECUDA, "cannot allocate the pinned staging buffer");
    h->stage_len = n;
  }
  if (!h->ev_stage && cudaEventCreateWithFlags(&h->ev_stage, cudaEventDisableTiming) != cudaSuccess) return fail_h(LLQ_ECUDA, "cudaEventCreate failed");
  // the previous host refresh's copy must have left the staging buffer before it is overwritten: the only host wait
  if (h->staged && cudaEventSynchronize(h->ev_stage) != cudaSuccess) return fail_h(LLQ_ECUDA, "staging event failed");
  memcpy(h->h_stage, weights, bytes);
  if (cudaMemcpyAsync(h->d_w + dst, h->h_stage, bytes, cudaMemcpyHostToDevice, s) != cudaSuccess || cudaEventRecord(h->ev_stage, s) != cudaSuccess)
    return fail_h(LLQ_ECUDA, "weight upload failed");
  h->staged = true;
  return LLQ_OK;
}

template <int MODE>
int launch(llq_hier_policy_handle h, const float* d_obs, int64_t obs_ld, int32_t n, const uint8_t* d_done, float* d_state, float* d_actions,
           int32_t* d_codes, float* d_heading, const Sample& smp, void* stream) {
  if (cudaSetDevice(h->device) != cudaSuccess) return fail_h(LLQ_ECUDA, "cudaSetDevice failed");
  Net net{h->d_w, h->d_off};
  if (!h->attr_set) {
    if (cudaFuncSetAttribute(hier_policy_kernel<M_DET>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(Smem)) != cudaSuccess ||
        (h->train && cudaFuncSetAttribute(h->strategic ? hier_policy_kernel<M_TRAIN_SEPMC> : hier_policy_kernel<M_TRAIN>,
                                          cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(Smem)) != cudaSuccess))
      return fail_h(LLQ_ECUDA, "cudaFuncSetAttribute failed");
    h->attr_set = true;                                      // per handle = per device
  }
  hier_policy_kernel<MODE><<<(n + kRows - 1) / kRows, kThreads, sizeof(Smem), (cudaStream_t)stream>>>(net, h->strategic, d_obs, obs_ld, n, d_done, d_state,
                                                                                                    d_actions, d_codes, d_heading, smp);
  if (cudaGetLastError() != cudaSuccess) return fail_h(LLQ_ECUDA, "hier_policy_kernel launch failed");
  return LLQ_OK;
}

}  // namespace

extern "C" {

int llq_hier_policy_create(const float* weights, int64_t n_weights, const int32_t* offsets, int32_t n_roles, int32_t strategic, int32_t device,
                           llq_hier_policy_handle* out) {
  return create(weights, n_weights, offsets, n_roles, nullptr, 0, strategic, device, out);
}

int llq_hier_policy_create_train(const float* weights, int64_t n_weights, const int32_t* offsets, int32_t n_roles, const int32_t* value_offsets,
                                 int32_t n_value_roles, int32_t strategic, int32_t device, llq_hier_policy_handle* out) {
  if (strategic)
    return fail_h(LLQ_EUNSUPPORTED, "this entry creates training handles for the environmental level only; the strategic level's is "
                                    "llq_hier_policy_create_train_strategic (include/llq_policy.h)");
  if (!value_offsets) return fail_h(LLQ_EINVAL, "null argument");
  if (n_value_roles != LLQ_HIER_ROLES_VALUE) return fail_h(LLQ_EINVAL, "value-tower table has the wrong length (include/llq_policy.h)");
  return create(weights, n_weights, offsets, n_roles, value_offsets, LLQ_HIER_ROLES_VALUE, 0, device, out);
}

int llq_hier_policy_create_train_strategic(const float* weights, int64_t n_weights, const int32_t* offsets, int32_t n_roles,
                                           const int32_t* train_offsets, int32_t n_train_roles, int32_t device, llq_hier_policy_handle* out) {
  if (!train_offsets) return fail_h(LLQ_EINVAL, "null argument");
  if (n_train_roles != LLQ_HIER_ROLES_TRAIN_STRATEGIC) return fail_h(LLQ_EINVAL, "strategic training table has the wrong length (include/llq_policy.h)");
  return create(weights, n_weights, offsets, n_roles, train_offsets, LLQ_HIER_ROLES_TRAIN_STRATEGIC, 1, device, out);
}

int llq_hier_policy_destroy(llq_hier_policy_handle h) {
  if (!h) return LLQ_OK;
  cudaSetDevice(h->device);
  cudaFree(h->d_w); cudaFree(h->d_off); cudaFree(h->d_seg);
  if (h->h_stage) cudaFreeHost(h->h_stage);
  if (h->ev_stage) cudaEventDestroy(h->ev_stage);
  delete h;
  return LLQ_OK;
}

int llq_hier_policy_forward(llq_hier_policy_handle h, const float* d_obs, int64_t obs_ld, int32_t n, const uint8_t* d_done, float* d_state,
                            float* d_actions, int32_t* d_codes, float* d_heading, void* stream) {
  if (!h || !d_obs || !d_state || !d_actions) return fail_h(LLQ_EINVAL, "null argument");
  if (h->n_models) return fail_h(LLQ_EINVAL, "a pool handle steps with llq_hier_policy_forward_pool");
  if (h->train)
    return fail_h(LLQ_EINVAL, h->strategic ? "a strategic training handle steps with llq_hier_policy_forward_rec_strategic (its state rows are 192 floats)"
                                           : "a training handle steps with llq_hier_policy_forward_rec (its state rows are 128 floats)");
  if (n <= 0 || obs_ld < (h->strategic ? 965 : 916)) return fail_h(LLQ_EINVAL, "bad row count or row stride");
  return launch<M_DET>(h, d_obs, obs_ld, n, d_done, d_state, d_actions, d_codes, d_heading, Sample{}, stream);
}

int llq_hier_policy_forward_rec(llq_hier_policy_handle h, const float* d_obs, int64_t obs_ld, int32_t n, const uint8_t* d_done, float* d_state,
                                float* d_actions, int32_t* d_codes, float* d_values, float* d_neglogp, int64_t out_ld, uint64_t seed, uint64_t counter,
                                int64_t row_gid0, void* stream) {
  if (!h || !d_obs || !d_state || !d_actions) return fail_h(LLQ_EINVAL, "null argument");
  if (!h->train) return fail_h(LLQ_EINVAL, "not a training handle (llq_hier_policy_create_train)");
  if (h->strategic) return fail_h(LLQ_EINVAL, "a strategic training handle steps with llq_hier_policy_forward_rec_strategic");
  if (n <= 0 || obs_ld < 916 || out_ld < 1) return fail_h(LLQ_EINVAL, "bad row count or row stride");
  const Sample smp{d_values, d_neglogp, (long long)out_ld, (unsigned long long)seed, (unsigned long long)counter, (long long)row_gid0};
  return launch<M_TRAIN>(h, d_obs, obs_ld, n, d_done, d_state, d_actions, d_codes, nullptr, smp, stream);
}

int llq_hier_policy_forward_rec_strategic(llq_hier_policy_handle h, const float* d_obs, int64_t obs_ld, int32_t n, const uint8_t* d_done,
                                          float* d_state, float* d_actions, int32_t* d_codes, float* d_heading, float* d_values, float* d_neglogp,
                                          int64_t out_ld, uint64_t seed, uint64_t counter, int64_t row_gid0, void* stream) {
  if (!h || !d_obs || !d_state || !d_actions) return fail_h(LLQ_EINVAL, "null argument");
  if (!h->train || !h->strategic) return fail_h(LLQ_EINVAL, "not a strategic training handle (llq_hier_policy_create_train_strategic)");
  if (n <= 0 || obs_ld < 965 || out_ld < 1) return fail_h(LLQ_EINVAL, "bad row count or row stride");
  const Sample smp{d_values, d_neglogp, (long long)out_ld, (unsigned long long)seed, (unsigned long long)counter, (long long)row_gid0};
  return launch<M_TRAIN_SEPMC>(h, d_obs, obs_ld, n, d_done, d_state, d_actions, d_codes, d_heading, smp, stream);
}

int llq_hier_policy_create_pool(const float* weights, int64_t n_weights, const int32_t* offsets, int32_t n_models, int32_t max_rows, int32_t device,
                                llq_hier_policy_handle* out) {
  if (!weights || !offsets || !out) return fail_h(LLQ_EINVAL, "null argument");
  if (n_models < 1 || n_models > LLQ_HIER_POOL_MAX) return fail_h(LLQ_EINVAL, "n_models outside [1, LLQ_HIER_POOL_MAX]");
  if (max_rows <= 0) return fail_h(LLQ_EINVAL, "max_rows must be positive");
  std::vector<int> off((size_t)n_models * RV);
  for (size_t i = 0; i < off.size(); i++) {
    if (offsets[i] < 0 || offsets[i] >= n_weights) return fail_h(LLQ_EINVAL, "role offset outside the weight blob");
    off[i] = offsets[i];
  }
  llq_hier_policy_handle h = nullptr;
  const int rc = upload(weights, n_weights, off, 1, 0, device, &h);
  if (rc != LLQ_OK) return rc;
  h->n_models = n_models; h->max_rows = max_rows;
  h->regions_ok = pool_regions(offsets, n_models, n_weights, h->region, h->region_end);
  const std::vector<double> uniform(n_models, 1.0);
  h->cut = cutoffs(uniform.data(), n_models);
  const size_t ws = (size_t)n_models + 1 + ((size_t)(max_rows + kRows - 1) / kRows + n_models) * kRows;
  if (cudaMalloc(&h->d_seg, sizeof(int) * ws) != cudaSuccess) {
    llq_hier_policy_destroy(h);
    return fail_h(LLQ_ECUDA, "workspace allocation failed");
  }
  *out = h;
  return LLQ_OK;
}

int llq_hier_policy_set_pool_probs(llq_hier_policy_handle h, const double* probs, int32_t n) {
  if (!h || !probs) return fail_h(LLQ_EINVAL, "null argument");
  if (!h->n_models) return fail_h(LLQ_EINVAL, "not a pool handle (llq_hier_policy_create_pool)");
  if (n != h->n_models) return fail_h(LLQ_EINVAL, "one probability per model");
  double s = 0.0;
  for (int k = 0; k < n; k++) {
    if (!std::isfinite(probs[k]) || probs[k] < 0.0) return fail_h(LLQ_EINVAL, "probabilities must be finite and >= 0");
    s += probs[k];
  }
  if (!(s > 0.0) || !std::isfinite(s)) return fail_h(LLQ_EINVAL, "probabilities must have a finite positive sum");
  h->cut = cutoffs(probs, n);
  return LLQ_OK;
}

int llq_hier_policy_forward_pool(llq_hier_policy_handle h, const float* d_obs, int64_t obs_ld, int32_t n, const uint8_t* d_done, float* d_state,
                                 float* d_actions, int32_t* d_codes, float* d_heading, int32_t* d_model, float* d_model_rec, int64_t rec_ld,
                                 uint64_t seed, uint64_t counter, int64_t row_gid0, void* stream) {
  if (!h || !d_obs || !d_state || !d_actions || !d_model) return fail_h(LLQ_EINVAL, "null argument");
  if (!h->n_models) return fail_h(LLQ_EINVAL, "not a pool handle (llq_hier_policy_create_pool)");
  if (n <= 0 || n > h->max_rows) return fail_h(LLQ_EINVAL, "row count outside [1, max_rows]");
  if (obs_ld < 965 || (d_model_rec && rec_ld < 1)) return fail_h(LLQ_EINVAL, "bad row stride");
  if (cudaSetDevice(h->device) != cudaSuccess) return fail_h(LLQ_ECUDA, "cudaSetDevice failed");
  if (!h->attr_set) {
    if (cudaFuncSetAttribute(hier_pool_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(PoolSmem)) != cudaSuccess)
      return fail_h(LLQ_ECUDA, "cudaFuncSetAttribute failed");
    h->attr_set = true;
  }
  const int K = h->n_models;
  int* seg_cta = h->d_seg;
  int* seg_rows = h->d_seg + K + 1;
  hier_pool_assign_kernel<<<1, kAssignThreads, 0, (cudaStream_t)stream>>>(n, K, h->cut, d_done, d_model, d_model_rec, (long long)rec_ld,
                                                                         (unsigned long long)seed, (unsigned long long)counter, (long long)row_gid0,
                                                                         seg_cta, seg_rows);
  if (cudaGetLastError() != cudaSuccess) return fail_h(LLQ_ECUDA, "hier_pool_assign_kernel launch failed");
  // every segment ends within kRows - 1 pad entries: at most ceil(n / kRows) + K - 1 CTAs, fixed here without reading the segments back
  hier_pool_kernel<<<(n + kRows - 1) / kRows + K, kThreads, sizeof(PoolSmem), (cudaStream_t)stream>>>(h->d_w, h->d_off, K, seg_cta, seg_rows, d_obs,
                                                                                                      obs_ld, d_done, d_state, d_actions, d_codes,
                                                                                                      d_heading);
  if (cudaGetLastError() != cudaSuccess) return fail_h(LLQ_ECUDA, "hier_pool_kernel launch failed");
  return LLQ_OK;
}

int llq_hier_policy_set_weights(llq_hier_policy_handle h, const float* weights, int64_t n_weights, int32_t on_device, void* stream) {
  if (!h || !weights) return fail_h(LLQ_EINVAL, "null argument");
  if (h->n_models) return fail_h(LLQ_EINVAL, "a pool handle replaces one model at a time: llq_hier_policy_set_pool_model");
  if (n_weights != h->n_weights) return fail_h(LLQ_EINVAL, "weight blob length differs from the one given at create");
  return refresh(h, 0, weights, n_weights, on_device, stream);
}

int llq_hier_policy_set_pool_model(llq_hier_policy_handle h, int32_t k, const float* weights, int64_t n_weights, int32_t on_device,
                                   void* stream) {
  if (!h || !weights) return fail_h(LLQ_EINVAL, "null argument");
  if (!h->n_models) return fail_h(LLQ_EINVAL, "not a pool handle (llq_hier_policy_create_pool)");
  if (k < 0 || k >= h->n_models) return fail_h(LLQ_EINVAL, "model index outside [0, n_models)");
  if (!h->regions_ok) return fail_h(LLQ_EINVAL, "the pool's models share arrays: a model has no region of its own");
  if (n_weights != h->region_end[k] - h->region[k]) return fail_h(LLQ_EINVAL, "weight blob length differs from model k's region");
  return refresh(h, h->region[k], weights, n_weights, on_device, stream);
}

const char* llq_hier_policy_last_error(void) { return g_err_h.c_str(); }

}  // extern "C"
