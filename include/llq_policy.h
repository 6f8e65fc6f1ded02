/* llq_policy.h -- C ABI of the on-device PMC policy forward (SURVEY.md 8 row f2).
 *
 * Replaces, for the batched actor loop, the TensorFlow graph of the reference's primitive-level policy evaluated once per
 * env step in `PGAgent.step(obs, argmax=True)` (test_scripts/primitive_level/test_primitive_level_env.py:75-88):
 *   networks/legged_robot/pmc_net/pmc_net.py:33-58   vq_encoder / decoder (fully connected, ReLU)
 *   networks/legged_robot/pmc_net/pmc_net.py:99-114  llc: prop 135 -> 64, z 32 -> 32, concat -> 256 -> 256 -> 12 (mean)
 *   networks/legged_robot/pmc_net/pmc_net.py:130-137 running-mean normalisation, clip to +-5 (networks/layers.py:55)
 *   networks/legged_robot/pmc_net/pmc_net.py:155-171 nearest code of the 32 x 256 codebook
 * The observation rows are read in place from the engine's device buffer (or a trajectory slab: `obs_ld` floats per row) and
 * the 12 actions per env are written to device memory that llq_step_ex(LLQ_IO_DEVICE) consumes: no host round trip.
 *
 * `weights`: the 28 arrays of a shipped *.model file, fp32, concatenated in their stored order:
 *   0-3   prop_mean[135] prop_std[135] future_mean[72] future_std[72]
 *   4-9   value head W1[207x256] b1[256] W2[256x256] b2[256] W3[256x1] b3[1]   (tanh; pmc_net.py:139-144)
 *   10-15 enc W1[207x256] b1[256] W2[256x256] b2[256] W3[256x32] b3[32]          16 codebook[32x256]
 *   17-20 prop_embed W[135x64] b[64], z_embed W[32x32] b[32]
 *   21-26 dec W1[96x256] b1[256] W2[256x256] b2[256] W3[256x12] b3[12]           27 logstd[12]
 * All matrices row major [in][out] as TensorFlow stores them. */
#ifndef LLQ_POLICY_H
#define LLQ_POLICY_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define LLQ_POLICY_N_WEIGHTS 358647   /* total floats of the list above */

typedef struct llq_policy* llq_policy_handle;

/* Uploads the weights to `device` and packs them there; returns once the handle is ready.  Returns 0 or a negative LLQ_E* code (llq.h); message via llq_policy_last_error(). */
int llq_policy_create(const float* weights, int64_t n_weights, int32_t device, llq_policy_handle* out);
int llq_policy_destroy(llq_policy_handle h);
/* actions[n,12] = mean action for obs[n, >=207] (device pointers; obs_ld = row stride in floats); `codes` (int32[n], device,
 * nullable) receives the selected codebook index.  Asynchronous on `stream` (a cudaStream_t, 0 = the default stream). */
int llq_policy_forward(llq_policy_handle h, const float* d_obs, int64_t obs_ld, int32_t n, float* d_actions, int32_t* d_codes, void* stream);
/* Full actor step for rollouts: as llq_policy_forward, plus
 *   d_values  (float[n], device, nullable): the value head's V(obs)  -> PMCInputs.V (pmc_net_data.py:7-16);
 *   d_neglogp (float[n], device, nullable): when given, d_actions receives a SAMPLE a = mean + exp(logstd) * eps of the diagonal
 *     Gaussian head (agent.step(argmax=False); pmc_net.py:107-113) and d_neglogp its -log p(a) = 0.5 sum eps^2 + sum logstd +
 *     6 log(2 pi) -> PMCInputs.neglogp; eps ~ N(0,1) from Philox4x32-10 keyed by `seed`, counter (row, draw, `counter`): pass a
 *     different `counter` every step.  NULL: d_actions is the mean (argmax=True). */
int llq_policy_forward_ex(llq_policy_handle h, const float* d_obs, int64_t obs_ld, int32_t n, float* d_actions, int32_t* d_codes,
                          float* d_values, float* d_neglogp, uint64_t seed, uint64_t counter, void* stream);
/* Record variant for the rollout worker (SURVEY 8e/f3: the kernels write the whole trajectory record): as llq_policy_forward_ex, but
 * value and -log p of row i go to d_values[i * out_ld] / d_neglogp[i * out_ld] (out_ld = the slab's row stride puts them straight into
 * the value / neglogp columns of a [N, 223] record row), and the Gaussian noise is keyed by the GLOBAL row row_gid0 + i so that
 * shards with equal seeds draw different noise (one actor process per shard in the reference draws from its own np.random). */
int llq_policy_forward_rec(llq_policy_handle h, const float* d_obs, int64_t obs_ld, int32_t n, float* d_actions, int32_t* d_codes,
                           float* d_values, float* d_neglogp, int64_t out_ld, uint64_t seed, uint64_t counter, int64_t row_gid0, void* stream);
/* Model refresh (a training actor following its learner): the handle takes a new 28-array blob of the same layout as at create.
 *   Ordering: asynchronous on `stream` (0 = the default stream); forwards queued on `stream` before the call see the old weights, forwards
 *     queued after it the new ones.  Nothing synchronises the device; forwards on OTHER streams are not ordered with the refresh.
 *   on_device = 0: `weights` is host memory, reusable as soon as the call returns: it is copied into a pinned staging buffer of the handle
 *     and uploaded with cudaMemcpyAsync on `stream` into the handle's raw blob (1.4 MB of device memory kept since create).  A second
 *     host refresh waits on the host (an event) until the previous upload has left the staging buffer: the only host wait, and only when
 *     two refreshes are closer together than one copy.
 *   on_device = 1: `weights` is device memory on the handle's device (e.g. a blob broadcast by the learner rank); host memory or another
 *     device returns LLQ_EINVAL.  The caller keeps it alive until the refresh has run on `stream`.
 *   The forward reads an image of the blob in MMA B-fragment order; the refresh rebuilds it in place with the same pack kernel as
 *   llq_policy_create (a pure permutation with zero padding).  Null arguments, a wrong length or a bad on_device return LLQ_EINVAL
 *   before the device is touched. */
int llq_policy_set_weights(llq_policy_handle h, const float* weights, int64_t n_weights, int32_t on_device, void* stream);
const char* llq_policy_last_error(void);

/* ---- environmental- and strategic-level policies (csrc/llq_policy_hier.cu): conv encoders + layer-norm LSTMs + the frozen
 * primitive-level decoder, one CTA per observation row, fp32 on the CUDA cores.  Replaces `PGAgent.step(obs, argmax=True)` of
 * test_scripts/environmental_level/test_environmental_level_env.py:95-100 and test_scripts/strategic_level/test_strategic_level_env.py:96
 * (mean heading, argmax code, mean action) for a whole batch of envs, and at both levels also the actor step of a training rollout
 * (environmental: sampled code, -log p, V, llq_hier_policy_forward_rec; strategic: sampled heading, -log p, V,
 * llq_hier_policy_forward_rec_strategic); nets: networks/legged_robot/epmc_net/epmc_net.py:86-177,
 * networks/legged_robot/sepmc_net/sepmc_net.py:122-203, networks/legged_robot/pmc_net/pmc_net.py:99-112.
 * `weights`: all arrays of the shipped *.model file, fp32, concatenated; `offsets[role]`: start of the array that plays `role`
 * (the host-side table is lifelike_agility_and_play_b200/policy_epmc.py::hier_role_arrays):
 *   0 prop mean, 1 prop std | code controller: 2-3 prop embed W b, 4-31 usr_cmd_encoder (2-D map 8, lidar 8, front map 8, target fc 2,
 *   fusion fc 2), 32-33 embed, 34-42 LSTM (wx wh b beta_x gamma_x beta_h gamma_h beta_c gamma_c), 43-44 logits, 45 codebook,
 *   46-55 low-level controller | heading controller (strategic level only): 56-57 prop embed, 58-83 perception encoder (24 + fusion fc 2),
 *   84-87 game-vector fc x 2, 88-89 embed, 90-98 LSTM, 99-100 heading fc. */
#define LLQ_HIER_ROLES_MLC 56
#define LLQ_HIER_ROLES_ALL 101
/* The value tower of the environmental level, arrays 2-46 of environmental_level_*.model, as its own table (its 45 entries next to
 * the 56 of the code controller would be indistinguishable from the strategic level's 101 by length):
 *   0-1 prop fc W b (135 -> 128), 2-29 usr_cmd_encoder (as roles 4-31), 30-31 command fc (64 -> 128), 32-33 fc (256 -> 256),
 *   34-42 LSTM (as roles 34-42), 43-44 value fc (32 -> 1, linear). */
#define LLQ_HIER_ROLES_VALUE 45
/* The strategic level's training table: its value tower, arrays 2-50 of strategic_level.model, then the heading logstd (array 96, (1, 1),
 * the one Gaussian parameter of the heading-controller block 51-96):
 *   0-1 prop fc W b (135 -> 128), 2-25 perception encoders (2-D map 8, lidar 8, front map 8; as roles 58-81), 26-27 perception fusion
 *   fc (88 -> 64), 28-29 perception fc (64 -> 128), 30-35 game-vector fc x 3 (29 -> 64 -> 64 -> 128), 36-37 concatenation fc (384 -> 256,
 *   input [prop | perception | game] as the heading controller's), 38-46 LSTM (as roles 34-42), 47-48 value fc (32 -> 1, linear),
 *   49 heading logstd.  All fully connected layers but the last take a ReLU. */
#define LLQ_HIER_ROLES_TRAIN_STRATEGIC 50
typedef struct llq_hier_policy* llq_hier_policy_handle;
int llq_hier_policy_create(const float* weights, int64_t n_weights, const int32_t* offsets, int32_t n_roles, int32_t strategic, int32_t device,
                           llq_hier_policy_handle* out);
/* Training handle of the environmental level (for llq_hier_policy_forward_rec): as llq_hier_policy_create with strategic = 0, plus
 * `value_offsets[LLQ_HIER_ROLES_VALUE]` (n_value_roles must equal it).  strategic != 0 returns LLQ_EUNSUPPORTED: the strategic level's
 * training handle comes from llq_hier_policy_create_train_strategic. */
int llq_hier_policy_create_train(const float* weights, int64_t n_weights, const int32_t* offsets, int32_t n_roles, const int32_t* value_offsets,
                                 int32_t n_value_roles, int32_t strategic, int32_t device, llq_hier_policy_handle* out);
/* Training handle of the strategic level (for llq_hier_policy_forward_rec_strategic): `offsets` is the 101-role table of
 * llq_hier_policy_create at the strategic level, `train_offsets[LLQ_HIER_ROLES_TRAIN_STRATEGIC]` the table above (n_train_roles must
 * equal it). */
int llq_hier_policy_create_train_strategic(const float* weights, int64_t n_weights, const int32_t* offsets, int32_t n_roles,
                                           const int32_t* train_offsets, int32_t n_train_roles, int32_t device, llq_hier_policy_handle* out);
int llq_hier_policy_destroy(llq_hier_policy_handle h);
/* d_actions[n,12] = mean action for d_obs[n, >= 916 (environmental) / 965 (strategic)] (device pointers, obs_ld = row stride in floats).
 * d_state [n, 64 / 128] floats: the LSTM states ([c, h] of the heading LSTM first at the strategic level), updated in place; rows whose
 * d_done[i] != 0 (uint8, nullable: the done flags of the step that produced these observations) start from a zero state.
 * d_codes (int32[n]) / d_heading (float[n], strategic level) are optional outputs.  Asynchronous on `stream`. */
int llq_hier_policy_forward(llq_hier_policy_handle h, const float* d_obs, int64_t obs_ld, int32_t n, const uint8_t* d_done, float* d_state,
                            float* d_actions, int32_t* d_codes, float* d_heading, void* stream);
/* Actor step of a training rollout at the environmental level (agent.step(argmax=False)), on a handle from
 * llq_hier_policy_create_train; llq_hier_policy_forward refuses such a handle.  As llq_hier_policy_forward, plus:
 *   the code is SAMPLED from the 256-way head by Gumbel-max, code = argmax_j (logit_j - log(-log u_j)) (first index on ties), with
 *     u = min((r + 1/2) 2^-32, 0.99999994f) in fp32 and r from Philox4x32-10, counter (low 32 bits of row_gid0 + i, q, `counter` lo,
 *     `counter` hi), key (`seed` lo, `seed` hi), q = 0..63 giving the draws of logits 4q..4q+3 -- keyed by the GLOBAL row as in
 *     llq_policy_forward_rec; pass a different `counter` every step.  d_actions is the decoder's action on the sampled code, and
 *     d_codes (int32[n], nullable) receives the sampled code;
 *   d_values[i * out_ld] (nullable): V of the value tower;  d_neglogp[i * out_ld] (nullable): -log p of the sampled code,
 *     m + log sum_j exp(logit_j - m) - logit_code with m the largest logit;  out_ld = the slab's row stride puts both into a record row;
 *   d_state [n, 128]: [c, h] of the code LSTM, then [c, h] of the value LSTM; both halves start from zero where d_done[i] != 0. */
int llq_hier_policy_forward_rec(llq_hier_policy_handle h, const float* d_obs, int64_t obs_ld, int32_t n, const uint8_t* d_done, float* d_state,
                                float* d_actions, int32_t* d_codes, float* d_values, float* d_neglogp, int64_t out_ld, uint64_t seed,
                                uint64_t counter, int64_t row_gid0, void* stream);
/* Actor step of a training rollout at the strategic level, on a handle from llq_hier_policy_create_train_strategic (the other entries
 * refuse such a handle, this one refuses every other handle and obs_ld < 965).  The heading is the level's action:
 *   a = mu + exp(logstd) eps, eps = sqrt(-2 log u0) cos(2 pi u1) with u0 = min((r.x + 1/2) 2^-32, 0.99999994f) and u1 = r.y 2^-32 in fp32,
 *     r from Philox4x32-10 with counter (low 32 bits of row_gid0 + i, 64, `counter` lo, `counter` hi) and key (`seed` lo, `seed` hi)
 *     (q = 64: apart from the Gumbel draws q = 0..63 of llq_hier_policy_forward_rec); pass a different `counter` every step;
 *   d_heading[i * out_ld] (nullable): the RAW a;  d_neglogp[i * out_ld] (nullable): its -log p = 0.5 eps^2 + logstd + 0.5 log(2 pi), fp32;
 *   d_values[i * out_ld] (nullable): V of the strategic value tower;
 *   the frozen code controller receives clip(a, +-3.14159265f), as in llq_hier_policy_forward, and takes the ARGMAX code (d_codes, int32[n],
 *     nullable); d_actions [n, 12] (contiguous) is the decoder's mean action on that code;
 *   d_state [n, 192]: [c, h] of the heading LSTM, of the code LSTM, then of the value LSTM; all three start from zero where d_done[i] != 0
 *     (d_done nullable). */
int llq_hier_policy_forward_rec_strategic(llq_hier_policy_handle h, const float* d_obs, int64_t obs_ld, int32_t n, const uint8_t* d_done,
                                          float* d_state, float* d_actions, int32_t* d_codes, float* d_heading, float* d_values, float* d_neglogp,
                                          int64_t out_ld, uint64_t seed, uint64_t counter, int64_t row_gid0, void* stream);
/* ---- opponent pool: K deterministic strategic-level models in one handle, every row run with its own model in one launch (a league
 * actor draws its frozen opponent per game; this is that draw for a whole batch of pairs).  A pool handle is refused by the other
 * forward entries and is single-owner: it holds one workspace, so two streams must not run llq_hier_policy_forward_pool on it at once.
 * Create: `weights` holds all K models; `offsets` [n_models * LLQ_HIER_ROLES_ALL], model k's 101-role table of llq_hier_policy_create
 * (strategic level) at offsets + k * LLQ_HIER_ROLES_ALL, absolute into `weights`; 1 <= n_models <= LLQ_HIER_POOL_MAX; `max_rows` bounds
 * n of every forward.  Null arguments, a bad count or an offset outside the blob return LLQ_EINVAL before the device is touched.  The
 * draw probabilities start uniform. */
#define LLQ_HIER_POOL_MAX 64
int llq_hier_policy_create_pool(const float* weights, int64_t n_weights, const int32_t* offsets, int32_t n_models, int32_t max_rows, int32_t device,
                                llq_hier_policy_handle* out);
/* Draw probabilities of the next forwards (n must equal n_models; every entry finite and >= 0, their sum > 0; else LLQ_EINVAL): the
 * host forms, in fp64, cum_k = p_0 + ... + p_k summed in order and the cutoffs t_k = floor(cum_k / cum_{K-1} * 2^32), t_{K-1} = 2^32; a
 * model with p = 0 is never drawn.  The cutoffs go to the next launch by value: no device copy, so a call between two steps is safe. */
int llq_hier_policy_set_pool_probs(llq_hier_policy_handle h, const double* probs, int32_t n);
/* One step of every row's model, on a pool handle (n <= max_rows, obs_ld >= 965).  First the draw: every row with d_done[i] != 0
 * (d_done nullable: no draws) gets d_model[i] = the smallest k with r < t_k, r = word x of Philox4x32-10 with counter (low 32 bits
 * of row_gid0 + i, 65, `counter` lo, `counter` hi) and key (`seed` lo, `seed` hi) (q = 65: apart from the Gumbel draws q = 0..63 and
 * the heading q = 64 of the training entries).  d_model (int32[n], device) is the caller's and is read by every call: rows keep their
 * model until they draw.  d_model_rec[i * rec_ld] (nullable) receives (float)d_model[i], or -1 outside [0, K), on every call.
 * Then, as llq_hier_policy_forward with model d_model[i] for row i: d_state [n, 128], d_actions [n, 12], d_codes, d_heading (both
 * nullable); a drawn row has d_done[i] != 0, so its state starts from zero.  A row whose model lies outside [0, K) is left untouched. */
int llq_hier_policy_forward_pool(llq_hier_policy_handle h, const float* d_obs, int64_t obs_ld, int32_t n, const uint8_t* d_done, float* d_state,
                                 float* d_actions, int32_t* d_codes, float* d_heading, int32_t* d_model, float* d_model_rec, int64_t rec_ld,
                                 uint64_t seed, uint64_t counter, int64_t row_gid0, void* stream);
/* Model refresh of a hierarchical handle (deterministic, environmental training or strategic training; a pool handle is refused and
 * pointed to llq_hier_policy_set_pool_model): the handle keeps the blob as given at create and its role tables hold offsets into it, so
 * the refresh is one copy of a blob of the same architecture and file layout (n_weights must equal the length given at create; the
 * role tables stay).  Ordering, on_device and the staging wait are those of llq_policy_set_weights.  The LSTM states are the caller's
 * and are not touched: a row continues its episode with the new weights. */
int llq_hier_policy_set_weights(llq_hier_policy_handle h, const float* weights, int64_t n_weights, int32_t on_device, void* stream);
/* Replaces model k (0 <= k < n_models; K is fixed at create) of a pool handle.  Model k's region of the pool blob runs from its
 * smallest role offset to the next larger model start (the smallest role offset of another model), or to the end of the blob; it is
 * computed at create.  n_weights must equal the region's length and the new model must be laid out like the one it replaces
 * (policy_epmc.DeviceOpponentPool lays every model out alike).  LLQ_EINVAL: k out of range, not a pool handle, or a pool whose models
 * share arrays (two models starting at the same float, or an array of model k starting outside its region).  Ordering and sources as
 * llq_hier_policy_set_weights.  Rows whose current game is against model k continue that game with the new weights and the state they
 * already carry; draws are not touched.  To grow a league, create the pool with the capacity needed, give the unused models probability
 * 0 (llq_hier_policy_set_pool_probs) and fill them later. */
int llq_hier_policy_set_pool_model(llq_hier_policy_handle h, int32_t k, const float* weights, int64_t n_weights, int32_t on_device,
                                   void* stream);
const char* llq_hier_policy_last_error(void);

/* ---- the learner seat of a strategic-level trajectory slab (csrc/llq_seat_pack.cu), for the hand-over of unrolls to the learner rank:
 * d_out [steps, pairs, 984] = the seat-0 rows d_slab[t, 2p] of a [steps, 2 pairs, 984] fp32 slab (row 2p of a step is the learning robot
 * of pair p, row 2p + 1 its opponent), a bit-exact copy in 16-byte vectors; both contiguous.  Asynchronous on `stream` (0 = the default
 * stream) of the pointers' device.  LLQ_EINVAL before the device is touched: a null pointer, a pointer that is not 16-byte aligned,
 * steps or pairs < 1 or too large for one launch, an output overlapping the slab; then LLQ_EINVAL for pointers that are not device
 * memory of one device.  Message via llq_seat_pack_last_error(). */
#define LLQ_SEPMC_RECORD 984
int llq_seat_pack(const float* d_slab, float* d_out, int64_t steps, int64_t pairs, void* stream);
const char* llq_seat_pack_last_error(void);

#ifdef __cplusplus
}
#endif
#endif
