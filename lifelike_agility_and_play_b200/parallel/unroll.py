"""TLeague-format unrolls from a gathered trajectory slab (SURVEY 8 row f3).

The reference's actor hands a finished unroll of ONE environment to the learner as the tuple
`(model_key, flat fp32 array, infos, shapes)` (learning/actors/distill_actor.py:164-167): every time step's record is
flattened leaf by leaf, all steps are concatenated into one 1-D array, and `shapes` holds the leaf shapes of one step so
that the learner's data server can restore the structure.  For the PMC policy-gradient learner the record is `PMCInputs`
(networks/legged_robot/pmc_net/pmc_net_data.py:7-16; placeholders pmc_net.py:60-96):

    X = OrderedDict(prop (99,), prop_a (36,), future (72,))   observation *before* the action (PLE:117-124)
    A (12,)   neglogp ()   discount ()   r (1,)   R (1,)   V (1,)   flatparam (24,) = mean | logstd

`discount` is gamma while the episode runs and 0 on the step that ended it; `R` is the lambda-return the reference learner
also builds for its ppo2 loss (pmc_net.py:213-224: `multistep_forward_view(reward, discounts, vpred[1:], lambda_)`):

    R_t = r_t + discount_t * ((1 - lam) * V_{t+1} + lam * R_{t+1}),     R_T = V_T (bootstrap)

with gamma = lam = 0.95 in the shipped training script (train_scripts/example_pmc_train.sh:21-22).

Here the rollout engine produces `[T, N, 223]` slabs (parallel/trajectory.py: obs 207 | action 12 | reward | done | neglogp |
value); this module turns a slab into the N per-environment tuples.  The return recursion runs as torch ops on whatever
device the slab lives on (a scan over T vectorised over the N environments); the flattening is a host-side reshape.
"""
from collections import OrderedDict

import numpy as np
import torch

from .trajectory import (ACT_DIM, COL_ACTION, COL_DONE, COL_NEGLOGP, COL_REWARD, COL_VALUE, HCOL_CODE, HCOL_DONE, HCOL_NEGLOGP, HCOL_REWARD,
                         HCOL_VALUE, HIER_TRAJ_WIDTH, OBS_DIM, SCOL_CODE, SCOL_DONE, SCOL_HEADING, SCOL_NEGLOGP, SCOL_OPPONENT, SCOL_REWARD,
                         SCOL_VALUE, SEPMC_TRAJ_WIDTH, TRAJ_WIDTH)

OBS_LEAVES = OrderedDict([("prop", 99), ("prop_a", 36), ("future", 72)])        # PLE:117-124
# leaf order of a flattened PMCInputs record (namedtuple order, the observation dict in key-insertion order)
RECORD_SHAPES = ((99,), (36,), (72,), (ACT_DIM,), (), (), (1,), (1,), (1,), (2 * ACT_DIM,))
RECORD_WIDTH = OBS_DIM + ACT_DIM + 5 + 2 * ACT_DIM                              # 248 floats per time step
GAMMA, LAM, LOGSTD_INIT = 0.95, 0.95, -2.0                                      # example_pmc_train.sh:21-22, pmc_net_data.py:93


def lambda_returns(reward, discount, value, bootstrap_value, lam=LAM):
    """R_t = r_t + discount_t * ((1-lam) V_{t+1} + lam R_{t+1}) over the leading (time) axis; all inputs `[T, N]`,
    `bootstrap_value` `[N]` = V of the observation that follows the slab's last step."""
    T = reward.shape[0]
    out = torch.empty_like(reward)
    nxt_v, nxt_r = bootstrap_value, bootstrap_value
    for t in range(T - 1, -1, -1):
        nxt_r = reward[t] + discount[t] * ((1.0 - lam) * nxt_v + lam * nxt_r)
        out[t] = nxt_r
        nxt_v = value[t]
    return out


def slab_records(slab, bootstrap_value=None, gamma=GAMMA, lam=LAM, flatparam=None, logstd=LOGSTD_INIT):
    """`[T, N, 223]` slab -> `[N, T, 248]` float32 records in PMCInputs leaf order (on the slab's device)."""
    assert slab.dim() == 3 and slab.shape[2] == TRAJ_WIDTH, "expected a [T, N, %d] trajectory slab" % TRAJ_WIDTH
    T, N, _ = slab.shape
    r, done, v = slab[:, :, COL_REWARD], slab[:, :, COL_DONE], slab[:, :, COL_VALUE]
    discount = gamma * (1.0 - done)
    if bootstrap_value is None:
        bootstrap_value = v[-1]
    ret = lambda_returns(r, discount, v, bootstrap_value.to(slab.dtype), lam)
    rec = torch.empty((N, T, RECORD_WIDTH), dtype=torch.float32, device=slab.device)
    c = OBS_DIM + ACT_DIM
    rec[:, :, :c] = slab[:, :, :c].transpose(0, 1)
    rec[:, :, c + 0] = slab[:, :, COL_NEGLOGP].t()
    rec[:, :, c + 1] = discount.t()
    rec[:, :, c + 2] = r.t()
    rec[:, :, c + 3] = ret.t()
    rec[:, :, c + 4] = v.t()
    if flatparam is None:       # deterministic head: mean = the action taken, log-std at its initial value
        rec[:, :, c + 5:c + 5 + ACT_DIM] = slab[:, :, COL_ACTION:COL_ACTION + ACT_DIM].transpose(0, 1)
        rec[:, :, c + 5 + ACT_DIM:] = logstd
    else:
        rec[:, :, c + 5:] = flatparam.transpose(0, 1)
    return rec


# observation leaves of the environmental level (PGE:129-137), in the order of its 916 observation columns
HIER_OBS_LEAVES = OrderedDict([("prop", (99,)), ("prop_a", (36,)), ("percep_2d", (25, 13)), ("percep_1d", (128,)), ("percep_front", (25, 13)),
                               ("target", (3,))])


def _recurrent_records(rows, leaves, actions, cols, initial_state, first_mask, bootstrap_value, gamma, lam):
    """Learner tensors of the learner's `rows` [T, N, width] of a recurrent unroll, in order: the observation `leaves` [T, N, *leaf], the
    level's `actions` ((name, [T, N] tensor) pairs), `neglogp`, `discount`, `r`, `V`, `R` (lambda-returns), `M` (the mask each forward
    received) and `S` = `initial_state`; `cols` = the record's (neglogp, reward, done, value) columns."""
    T, N = rows.shape[:2]
    out = OrderedDict()
    c = 0
    for name, shape in leaves.items():
        k = int(np.prod(shape))
        out[name] = rows[:, :, c:c + k].reshape(T, N, *shape)
        c += k
    out.update(actions)
    neglogp, r, done, v = (rows[:, :, k] for k in cols)
    discount = gamma * (1.0 - done)
    out["neglogp"], out["discount"], out["r"], out["V"] = neglogp, discount, r, v
    out["R"] = lambda_returns(r, discount, v, bootstrap_value.to(rows.dtype), lam)
    mask = torch.empty((T, N), dtype=rows.dtype, device=rows.device)
    mask[0] = (first_mask != 0).to(rows.dtype)
    mask[1:] = (done[:-1] != 0).to(rows.dtype)
    out["M"] = mask
    out["S"] = initial_state
    return out


def hier_slab_records(slab, initial_state, first_mask, bootstrap_value, gamma=GAMMA, lam=LAM):
    """Learner tensors of an environmental-level unroll (`HierRolloutWorker.finish_unroll()`), on the slab's device, named:
    the observation leaves [T, N, *leaf], `A_Z` [T, N] int64 (the sampled code), `neglogp`, `discount` = gamma (1 - done), `r`,
    `V`, `R` (lambda-returns, bootstrapped with V(observation T)), `M` [T, N] = the mask each forward received (M[0] = first_mask,
    M[t] = done[t-1]) -- all [T, N] float32 -- and `S` [N, 128], the recurrent state the unroll started from (code LSTM [c, h], then
    value LSTM [c, h])."""
    assert slab.dim() == 3 and slab.shape[2] == HIER_TRAJ_WIDTH, "expected a [T, N, %d] trajectory slab" % HIER_TRAJ_WIDTH
    return _recurrent_records(slab, HIER_OBS_LEAVES, [("A_Z", slab[:, :, HCOL_CODE].to(torch.int64))],
                              (HCOL_NEGLOGP, HCOL_REWARD, HCOL_DONE, HCOL_VALUE), initial_state, first_mask, bootstrap_value, gamma, lam)


# observation leaves of the strategic level (CTG:111-124), in the order of its 965 observation columns
SEPMC_OBS_LEAVES = OrderedDict([("prop", (99,)), ("prop_a", (36,)), ("percept_2d", (25, 13)), ("percept_1d", (128,)), ("percept_front", (25, 13)),
                                ("percept_vec", (5,)), ("oppo_info", (15,)), ("oppo_info_cheat", (15,)), ("flag_info", (7,)),
                                ("flag_info_cheat", (7,)), ("with_flag", (2,)), ("control_spd", (1,))])


def sepmc_slab_records(slab, initial_state, first_mask, bootstrap_value, gamma=GAMMA, lam=LAM, with_opponent=False, learner_seat_only=False):
    """Learner tensors of a strategic-level unroll (`SepmcRolloutWorker.finish_unroll()`) for the learning robot (seat 0: rows 0, 2, 4, ...
    of the `[T, 2P, 984]` slab), on the slab's device, named: the twelve observation leaves [T, P, *leaf] (CTG:111-124), `A_HLC` [T, P]
    (the raw sampled heading), `A_Z` [T, P] int64 (the argmax code), `neglogp` (of the heading), `discount` = gamma (1 - done), `r`, `V`,
    `R` (lambda-returns, bootstrapped with V(observation T)), `M` [T, P] = the mask each forward received (M[0] = first_mask, M[t] =
    done[t-1]) -- all [T, P] float32 but A_Z -- and `S` [P, 192], the recurrent state the unroll started from (heading, code and value
    LSTM, [c, h] each).  `with_opponent`: also `opponent` [T, P] int64 last, the index of the model seat 1 played in an opponent
    pool (for the league's per-opponent statistics; 0 against a single opponent).  `learner_seat_only`: `slab` holds the seat-0 records
    alone, `[T, P, 984]` (what `UnrollExchange(..., learner_seat_only=True)` gathers); the tensors are those of the full slab, bit for bit.
    P is the length of `first_mask`."""
    P = first_mask.shape[0]
    if learner_seat_only:
        assert slab.dim() == 3 and slab.shape[2] == SEPMC_TRAJ_WIDTH and slab.shape[1] == P, \
            "expected a [T, P, %d] learner-seat slab (P = len(first_mask) = %d)" % (SEPMC_TRAJ_WIDTH, P)
        s0 = slab
    else:
        assert slab.dim() == 3 and slab.shape[2] == SEPMC_TRAJ_WIDTH and slab.shape[1] == 2 * P, \
            "expected a [T, 2P, %d] trajectory slab (P = len(first_mask) = %d)" % (SEPMC_TRAJ_WIDTH, P)
        s0 = slab[:, 0::2]
    out = _recurrent_records(s0, SEPMC_OBS_LEAVES, [("A_HLC", s0[:, :, SCOL_HEADING]), ("A_Z", s0[:, :, SCOL_CODE].to(torch.int64))],
                             (SCOL_NEGLOGP, SCOL_REWARD, SCOL_DONE, SCOL_VALUE), initial_state, first_mask, bootstrap_value, gamma, lam)
    if with_opponent:
        out["opponent"] = s0[:, :, SCOL_OPPONENT].to(torch.int64)
    return out


def slab_to_unrolls(slab, model_key, infos=None, **kw):
    """The N tuples `(model_key, flat array, infos, shapes)` the reference actor would have pushed, one per environment
    (distill_actor.py:164-167).  `infos[i]` = list of the `info` dicts of env i's episodes that ended inside the slab."""
    rec = slab_records(slab, **kw).cpu().numpy()
    n = rec.shape[0]
    return [(model_key, rec[i].reshape(-1), list(infos[i]) if infos is not None else [], RECORD_SHAPES) for i in range(n)]


def unflatten_unroll(flat, shapes=RECORD_SHAPES):
    """Inverse of the flattening (what the learner's data server does with `shapes`): list over time of leaf lists."""
    sizes = [int(np.prod(s)) if len(s) else 1 for s in shapes]
    w = sum(sizes)
    assert flat.size % w == 0
    steps = flat.reshape(-1, w)
    out = []
    for row in steps:
        leaves, o = [], 0
        for s, k in zip(shapes, sizes):
            leaves.append(row[o:o + k].reshape(s))
            o += k
        out.append(leaves)
    return out
