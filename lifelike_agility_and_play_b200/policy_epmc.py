"""Host restatement (numpy) of the environmental-level policy's inference path, for evaluation runs on the vectorised engine
(SURVEY row f2 for EPMC; tools/statistical_pin_epmc.py).

Follows networks/legged_robot/epmc_net/epmc_net.py with the shipped actor configuration (train_scripts/example_epmc_train.sh:53-82:
llc_light, discrete_z, expert_lstm, lstm_layer_norm, append_hist_a, rms on the proprioception only):

* `usr_cmd_encoder` (epmc_net.py:120-135): target 3 -> 32 (ReLU) | `percep_2d_encoder` on the 25 x 13 height map (:86-94: 1x1 conv 4,
  4x4 stride 2, 2x2 stride 2, 2x2 -> 1 channel, all SAME + ReLU = the `tf.contrib.layers.conv2d` defaults) -> 28 | `percep_1d_encoder`
  on the 128 lidar rays (:109-117: periodic padding 4, conv1d 4 SAME, crop, two stride-2 convs, one to 1 channel) -> 32 | the same 2-D
  encoder with its own weights on the front map -> 28; concatenated (120) -> 64 (ReLU);
* `mlc_encoder` (:138-166): prop 135 -> 64, concat with the command embedding -> 256 (ReLU) -> LSTM(32, layer norm) -> 256 logits;
  the code index (argmax here, a categorical sample in the actor) selects a column of the primitive-level codebook (`mapping_z`,
  :169-177);
* `llc` (pmc_net.py:99-112): the frozen primitive-level decoder, prop 135 -> 64 | z 32 -> 32 -> 256 -> 256 -> 12.

The LSTM comes from `tpolicies` (TLeague's policy library, absent from the reference tree): restated from its published form --
`z = ln(x wx) + ln(h wh) + b`, gates `i, f, o, u`, `f = sigmoid(f + forget_bias)`, `h = o tanh(ln(c))`, state `[c, h]`, both zeroed
where the mask (episode start) is set -- with the variable order of the shipped files: wx, wh, b, then (beta, gamma) of the three layer
norms (x, h, c), as `tf.contrib.layers.layer_norm` creates them; the three additive vectors carry identical values in the shipped
files (same initialiser, same gradient), the two 128-vectors and the 32-vector with means 2.2 / 1.1 / 3.6 are the gains.  Nothing pins
this restatement bit for bit (no TensorFlow here); it is pinned behaviourally: the shipped Bullet-trained weights have to traverse the
corridors on the engine (DESIGN.md 6).

`weights` = the list of 102 arrays of a shipped ``environmental_level_*.model``:
0-1 prop running mean / std | 2-46 value tower (unused here except by `value`) | 47-48 prop embed | 49-76 command encoder |
77-78 embed | 79-87 LSTM | 88-89 logits | 90 codebook | 91-100 low-level controller | 101 logstd
"""
import ctypes as C

import numpy as np

from .policy import check_arrays, check_device_blob, is_tensor, keep_for_stream


def _same_pad(n, k, s):
    out = -(-n // s)
    total = max((out - 1) * s + k - n, 0)
    return out, total // 2, total - total // 2


def conv2d_same_relu(x, w, b, stride):
    """x [B, H, W, C], w [kh, kw, C, O] (TF layout), SAME padding, ReLU."""
    B, H, W, C = x.shape
    kh, kw, _, O = w.shape
    oh, pt, pb = _same_pad(H, kh, stride)
    ow, pl, pr = _same_pad(W, kw, stride)
    xp = np.pad(x, ((0, 0), (pt, pb), (pl, pr), (0, 0)))
    out = np.zeros((B, oh, ow, O), np.float32)
    for i in range(kh):
        for j in range(kw):
            patch = xp[:, i:i + (oh - 1) * stride + 1:stride, j:j + (ow - 1) * stride + 1:stride, :]
            out += patch @ w[i, j]
    return np.maximum(out + b, 0.0)


def conv1d_same_relu(x, w, b, stride):
    """x [B, W, C], w [k, C, O], SAME padding, ReLU."""
    return conv2d_same_relu(x[:, None], w[None], b, stride)[:, 0] if stride == 1 else \
        _conv1d_strided(x, w, b, stride)


def _conv1d_strided(x, w, b, stride):
    B, W, C = x.shape
    k, _, O = w.shape
    ow, pl, pr = _same_pad(W, k, stride)
    xp = np.pad(x, ((0, 0), (pl, pr), (0, 0)))
    out = np.zeros((B, ow, O), np.float32)
    for j in range(k):
        out += xp[:, j:j + (ow - 1) * stride + 1:stride, :] @ w[j]
    return np.maximum(out + b, 0.0)


def _ln(x, g, b, eps=1e-12):        # tf.contrib.layers.layer_norm: last axis, variance_epsilon 1e-12
    m = x.mean(1, keepdims=True)
    v = ((x - m) ** 2).mean(1, keepdims=True)
    return (x - m) / np.sqrt(v + eps) * g + b


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


class LnLstm:
    def __init__(self, w, forget_bias=1.0):
        self.wx, self.wh, self.b, self.bx, self.gx, self.bh, self.gh, self.bc, self.gc = w
        self.nh = self.wh.shape[0]
        self.forget_bias = forget_bias

    def step(self, x, state, mask):
        """x [B, nin], state [B, 2 nh] = [c, h], mask [B] (1 = the episode starts with this step)."""
        keep = (1.0 - mask)[:, None]
        c, h = state[:, :self.nh] * keep, state[:, self.nh:] * keep
        z = _ln(x @ self.wx, self.gx, self.bx) + _ln(h @ self.wh, self.gh, self.bh) + self.b
        i, f, o, u = np.split(z, 4, axis=1)
        c = _sigmoid(f + self.forget_bias) * c + _sigmoid(i) * np.tanh(u)
        h = _sigmoid(o) * np.tanh(_ln(c, self.gc, self.bc))
        return h, np.concatenate([c, h], axis=1).astype(np.float32)


class CommandEncoder:
    def __init__(self, w):
        """w = the arrays of one `usr_cmd_encoder` in creation order: percep_2d (8), percep_1d (8), percep_front (8), [vector feature
        (2),] fc (2) -- 28 with the vector feature (the target direction), 26 without (sepmc_net.py:149-173 before `target_info` exists)."""
        self.c2d, self.c1d, self.cfr = w[0:8], w[8:16], w[16:24]
        if len(w) == 28:
            self.wt, self.bt, self.wf, self.bf = w[24], w[25], w[26], w[27]
        else:
            assert len(w) == 26
            self.wt, self.bt, self.wf, self.bf = None, None, w[24], w[25]

    @staticmethod
    def _enc2d(x, w):
        e = x[..., None].astype(np.float32)
        e = conv2d_same_relu(e, w[0], w[1], 1)
        e = conv2d_same_relu(e, w[2], w[3], 2)
        e = conv2d_same_relu(e, w[4], w[5], 2)
        e = conv2d_same_relu(e, w[6], w[7], 1)
        return e.reshape(e.shape[0], -1)

    @staticmethod
    def _enc1d(x, w, k=4):
        p = np.concatenate([x[:, -k:], x, x[:, :k]], axis=1)[..., None].astype(np.float32)     # periodic padding (epmc_net.py:97-106)
        e = conv1d_same_relu(p, w[0], w[1], 1)[:, k:-k, :]
        e = conv1d_same_relu(e, w[2], w[3], 2)
        e = conv1d_same_relu(e, w[4], w[5], 2)
        e = conv1d_same_relu(e, w[6], w[7], 1)
        return e.reshape(e.shape[0], -1)

    def __call__(self, percep_2d, percep_1d, percep_front, target=None):
        parts = [self._enc2d(percep_2d, self.c2d), self._enc1d(percep_1d, self.c1d), self._enc2d(percep_front, self.cfr)]
        if self.wt is not None:
            parts = [np.maximum(target @ self.wt + self.bt, 0.0)] + parts
        e = np.concatenate(parts, axis=1)
        return np.maximum(e @ self.wf + self.bf, 0.0)


class EpmcPolicy:
    """Deterministic inference (argmax code, mean action) of the shipped environmental-level policy on [N, 916] engine observations."""

    def __init__(self, weights):
        w = [np.asarray(a, np.float32) for a in weights]
        assert len(w) == 102 and w[0].shape == (1, 135) and w[90].shape == (32, 256), "not an environmental-level model"
        self.mean, self.std = w[0], w[1]
        self.vf_fc1, self.vf_cmd, self.vf_fc2, self.vf_fc3 = (w[2], w[3]), CommandEncoder(w[4:32]), (w[32], w[33]), (w[34], w[35])
        self.vf_lstm, self.vf_out = LnLstm(w[36:45]), (w[45], w[46])
        self.prop_embed, self.cmd, self.embed = (w[47], w[48]), CommandEncoder(w[49:77]), (w[77], w[78])
        self.lstm, self.logits = LnLstm(w[79:88]), (w[88], w[89])
        self.codebook = w[90]
        self.llc_prop, self.llc_z = (w[91], w[92]), (w[93], w[94])
        self.dec = [(w[95], w[96]), (w[97], w[98]), (w[99], w[100])]
        self.logstd = w[101]
        self.nh = 32

    def initial_state(self, n):
        return np.zeros((n, 2 * self.nh), np.float32)

    @staticmethod
    def split(obs):
        o = np.asarray(obs, np.float32)
        return (o[:, 0:135], o[:, 135:460].reshape(-1, 25, 13), o[:, 460:588], o[:, 588:913].reshape(-1, 25, 13), o[:, 913:916])

    def value(self, obs, state, mask):
        """V(obs) of the value tower (arrays 2-46), state [N, 64] = [c, h] of its own LSTM, mask as in `act`.  Returns (V [N], new state).

        The wiring is restated from the array shapes with the code controller's conventions (the actor's value head of
        example_epmc_train.sh; epmc_net.py's value part is not in the reference tree):
            v1 = relu(p W2 + b3)                       135 -> 128   (p = the normalised, clipped prop)
            ce = usr_cmd_encoder(arrays 4-31)          target 3 -> 32 | 3 perception encoders 88 -> 120 -> 64
            v2 = relu(ce W32 + b33)                    64 -> 128
            v3 = relu([v1 | v2] W34 + b35)             256 -> 256   (the code controller's [prop | command] order)
            (c, h) = layer-norm LSTM(arrays 36-44)     state [c, h], zeroed where mask is set
            V  = h W45 + b46                           32 -> 1, linear
        Like the LSTM restatement above, nothing pins this against TensorFlow here: there is no TF, no shipped model file and no
        epmc_net.py value code in this tree.  It is the statement the device's training forward (llq_hier_policy_forward_rec) is
        checked against."""
        prop, p2d, p1d, pfr, tgt = self.split(obs)
        p = np.clip((prop - self.mean) / (self.std + 1e-8), -5.0, 5.0)
        v1 = np.maximum(p @ self.vf_fc1[0] + self.vf_fc1[1], 0.0)
        v2 = np.maximum(self.vf_cmd(p2d, p1d, pfr, tgt) @ self.vf_fc2[0] + self.vf_fc2[1], 0.0)
        v3 = np.maximum(np.concatenate([v1, v2], axis=1) @ self.vf_fc3[0] + self.vf_fc3[1], 0.0)
        h, state = self.vf_lstm.step(v3, state, np.asarray(mask, np.float32))
        return (h @ self.vf_out[0] + self.vf_out[1])[:, 0].astype(np.float32), state

    @staticmethod
    def gumbel(uniforms):
        """g = -log(-log u) of the Gumbel-max sample (fp64)."""
        return -np.log(-np.log(np.asarray(uniforms, np.float64)))

    def act(self, obs, state, mask, rng=None, return_code=False, uniforms=None, return_neglogp=False):
        """obs [N, 916] (prop 99 | prop_a 36 | percep_2d 325 | percep_1d 128 | percep_front 325 | target 3), state [N, 64] of the z-LSTM,
        mask [N] = 1 where the observation is the first of an episode.  `rng`: sample the code from the logits (the actor's
        behaviour) instead of the argmax; `uniforms` [N, 256] in (0, 1): sample it from these draws, code = argmax(logits + gumbel(u))
        (the device's training forward draws them from Philox, include/llq_policy.h).  Returns (action [N, 12], new state), then the
        code with `return_code`, then -log p of the code under the 256-way categorical with `return_neglogp`."""
        prop, p2d, p1d, pfr, tgt = self.split(obs)
        p = np.clip((prop - self.mean) / (self.std + 1e-8), -5.0, 5.0)
        pe = np.maximum(p @ self.prop_embed[0] + self.prop_embed[1], 0.0)
        ce = self.cmd(p2d, p1d, pfr, tgt)
        e = np.maximum(np.concatenate([pe, ce], axis=1) @ self.embed[0] + self.embed[1], 0.0)
        h, state = self.lstm.step(e, state, np.asarray(mask, np.float32))
        logits = h @ self.logits[0] + self.logits[1]
        if uniforms is not None:
            code = (logits + self.gumbel(uniforms)).argmax(1)
        elif rng is None:
            code = logits.argmax(1)
        else:
            g = -np.log(-np.log(rng.uniform(1e-12, 1.0, logits.shape)))
            code = (logits + g).argmax(1)
        z = self.codebook.T[code]
        a = np.maximum(p @ self.llc_prop[0] + self.llc_prop[1], 0.0)
        b = np.maximum(z @ self.llc_z[0] + self.llc_z[1], 0.0)
        x = np.concatenate([a, b], axis=1)
        x = np.maximum(x @ self.dec[0][0] + self.dec[0][1], 0.0)
        x = np.maximum(x @ self.dec[1][0] + self.dec[1][1], 0.0)
        act = (x @ self.dec[2][0] + self.dec[2][1]).astype(np.float32)
        out = (act, state) + ((code,) if return_code else ())
        if return_neglogp:
            lg = logits.astype(np.float64)
            m = lg.max(1)
            out += ((m - lg[np.arange(len(code)), code]) + np.log(np.exp(lg - m[:, None]).sum(1)),)
        return out


class SepmcPolicy:
    """Deterministic inference of the shipped strategic-level policy (networks/legged_robot/sepmc_net/sepmc_net.py, actor configuration
    of test_scripts/strategic_level/test_strategic_level_env.py:44-75) on [N, 965] engine observations: `hlc_encoder` (sepmc_net.py:122-146:
    prop 135 -> 64 | perception 88 -> 64 | game vector 29 -> 64 -> 64, concat 192 -> 256 -> LSTM(32) -> heading angle, clipped to +-pi),
    whose (cos, sin) joins the commanded speed as the `target_info` of the environmental-level encoder (`mlc_encoder`, :176-203) -> 256-way
    code -> the frozen primitive-level decoder.  `weights` = the 152 arrays of ``strategic_level.model``:
    0-1 rms | 2-50 value tower | 51-96 heading controller (96: the heading's logstd) | 97-139 code controller | 140 codebook |
    141-150 decoder | 151 logstd."""

    def __init__(self, weights):
        w = [np.asarray(a, np.float32) for a in weights]
        assert len(w) == 152 and w[83].shape == (192, 256) and w[140].shape == (32, 256), "not a strategic-level model"
        self.mean, self.std = w[0], w[1]
        self.vf_prop, self.vf_percept, self.vf_perc_fc = (w[2], w[3]), CommandEncoder(w[4:30]), (w[30], w[31])
        self.vf_game = [(w[32], w[33]), (w[34], w[35]), (w[36], w[37])]
        self.vf_cat, self.vf_lstm, self.vf_out = (w[38], w[39]), LnLstm(w[40:49]), (w[49], w[50])
        self.h_prop, self.h_percept = (w[51], w[52]), CommandEncoder(w[53:79])
        self.h_vec = [(w[79], w[80]), (w[81], w[82])]
        self.h_embed, self.h_lstm, self.h_mu, self.h_logstd = (w[83], w[84]), LnLstm(w[85:94]), (w[94], w[95]), w[96]
        self.m_prop, self.m_cmd, self.m_embed = (w[97], w[98]), CommandEncoder(w[99:127]), (w[127], w[128])
        self.m_lstm, self.logits = LnLstm(w[129:138]), (w[138], w[139])
        self.codebook = w[140]
        self.llc_prop, self.llc_z = (w[141], w[142]), (w[143], w[144])
        self.dec = [(w[145], w[146]), (w[147], w[148]), (w[149], w[150])]
        self.nh = 32

    def initial_state(self, n):
        return np.zeros((n, 4 * self.nh), np.float32)          # [c, h] of the heading LSTM, then of the code LSTM

    def _split(self, obs):
        o = np.asarray(obs, np.float32)
        prop, p2d, p1d, pfr = o[:, 0:135], o[:, 135:460].reshape(-1, 25, 13), o[:, 460:588], o[:, 588:913].reshape(-1, 25, 13)
        game = np.concatenate([o[:, 913:918], o[:, 918:933], o[:, 948:955], o[:, 962:964]], axis=1)      # percept_vec | oppo_info | flag_info | with_flag
        p = np.clip((prop - self.mean) / (self.std + 1e-8), -5.0, 5.0)
        return p, p2d, p1d, pfr, game, o[:, 964:965]

    def value(self, obs, state, mask):
        """V(obs) of the value tower (arrays 2-50), state [N, 64] = [c, h] of its own LSTM, mask as in `act`.  Returns (V [N], new state).

        The wiring is read off the array shapes with the heading controller's [prop | perception | game] order (the actor's value head of
        example_sepmc_train.sh; sepmc_net.py's value part is not in the reference tree):
            v1 = relu(p W2 + b3)                            135 -> 128
            v2 = relu(usr_cmd_encoder(arrays 4-29) W30 + b31)    perception 88 -> 64 (no target), then 64 -> 128
            v3 = game vector 29 -> 64 -> 64 -> 128          arrays 32-37, ReLU
            v4 = relu([v1 | v2 | v3] W38 + b39)             384 -> 256
            (c, h) = layer-norm LSTM(arrays 40-48)          state [c, h], zeroed where mask is set
            V  = h W49 + b50                                32 -> 1, linear
        Nothing pins this against TensorFlow here; it is the statement the device's strategic training forward
        (llq_hier_policy_forward_rec_strategic) is checked against."""
        p, p2d, p1d, pfr, game, _ = self._split(obs)
        relu = lambda x: np.maximum(x, 0.0)
        v1 = relu(p @ self.vf_prop[0] + self.vf_prop[1])
        v2 = relu(self.vf_percept(p2d, p1d, pfr) @ self.vf_perc_fc[0] + self.vf_perc_fc[1])
        v3 = game
        for W, b in self.vf_game:
            v3 = relu(v3 @ W + b)
        v4 = relu(np.concatenate([v1, v2, v3], axis=1) @ self.vf_cat[0] + self.vf_cat[1])
        h, state = self.vf_lstm.step(v4, state, np.asarray(mask, np.float32))
        return (h @ self.vf_out[0] + self.vf_out[1])[:, 0].astype(np.float32), state

    def act(self, obs, state, mask, return_aux=False, eps=None, return_neglogp=False):
        """obs [N, 965], state [N, 128] ([c, h] of the heading LSTM, then of the code LSTM), mask [N] = 1 where the observation is the
        first of an episode.  Returns (action [N, 12], new state), then (heading, code) with `return_aux`.  Without `eps` the heading is
        the mean, clipped to +-pi.  `eps` [N]: the heading is SAMPLED, a = mean + exp(logstd) eps (the training actor's behaviour; the
        device's training forward draws eps by Box-Muller from Philox, include/llq_policy.h); the code controller receives clip(a, +-pi),
        and the returned heading is the raw a; `return_neglogp` appends -log p(a) = 0.5 eps^2 + logstd + 0.5 log(2 pi)."""
        p, p2d, p1d, pfr, game, spd = self._split(obs)
        mask = np.asarray(mask, np.float32)
        relu = lambda x: np.maximum(x, 0.0)
        ge = relu(relu(game @ self.h_vec[0][0] + self.h_vec[0][1]) @ self.h_vec[1][0] + self.h_vec[1][1])
        e = relu(np.concatenate([relu(p @ self.h_prop[0] + self.h_prop[1]), self.h_percept(p2d, p1d, pfr), ge], axis=1) @ self.h_embed[0] + self.h_embed[1])
        hh, s_h = self.h_lstm.step(e, state[:, :2 * self.nh], mask)
        mu = hh @ self.h_mu[0] + self.h_mu[1]
        if eps is None:
            ang = head = np.clip(mu, -np.pi, np.pi)
        else:
            eps = np.asarray(eps, np.float64).reshape(-1, 1)
            ls = float(self.h_logstd.reshape(-1)[0])
            head = (mu + np.exp(ls) * eps).astype(np.float32)
            ang = np.clip(head, -np.float32(np.pi), np.float32(np.pi))
        tgt = np.concatenate([np.cos(ang), np.sin(ang), spd], axis=1).astype(np.float32)
        e2 = relu(np.concatenate([relu(p @ self.m_prop[0] + self.m_prop[1]), self.m_cmd(p2d, p1d, pfr, tgt)], axis=1) @ self.m_embed[0] + self.m_embed[1])
        hm, s_m = self.m_lstm.step(e2, state[:, 2 * self.nh:], mask)
        code = (hm @ self.logits[0] + self.logits[1]).argmax(1)
        z = self.codebook.T[code]
        x = np.concatenate([relu(p @ self.llc_prop[0] + self.llc_prop[1]), relu(z @ self.llc_z[0] + self.llc_z[1])], axis=1)
        x = relu(x @ self.dec[0][0] + self.dec[0][1])
        x = relu(x @ self.dec[1][0] + self.dec[1][1])
        act = (x @ self.dec[2][0] + self.dec[2][1]).astype(np.float32)
        new_state = np.concatenate([s_h, s_m], axis=1)
        out = (act, new_state) + ((head[:, 0], code) if return_aux else ())
        if return_neglogp:
            assert eps is not None, "-log p is that of a sampled heading: pass eps"
            out += (0.5 * eps[:, 0] ** 2 + ls + 0.5 * np.log(2.0 * np.pi),)
        return out


_ENC = [(1, 1, 1, 4), (4,), (4, 4, 4, 4), (4,), (2, 2, 4, 4), (4,), (2, 2, 4, 1), (1,), (4, 1, 4), (4,), (4, 4, 4), (4,), (4, 4, 4), (4,), (4, 4, 1), (1,),
        (1, 1, 1, 4), (4,), (4, 4, 4, 4), (4,), (2, 2, 4, 4), (4,), (2, 2, 4, 1), (1,)]
_ENC28, _ENC26 = _ENC + [(3, 32), (32,), (120, 64), (64,)], _ENC + [(88, 64), (64,)]
_LSTM = [(256, 128), (32, 128), (128,), (128,), (128,), (128,), (128,), (32,), (32,)]
_LLC = [(135, 64), (64,), (32, 32), (32,), (96, 256), (256,), (256, 256), (256,), (256, 12), (12,), (1, 12)]
# array shapes of the shipped files, in their stored order (environmental_level_*.model: 102 arrays, strategic_level.model: 152)
EPMC_SHAPES = ([(1, 135), (1, 135), (135, 128), (128,)] + _ENC28 + [(64, 128), (128,), (256, 256), (256,)] + _LSTM + [(32, 1), (1,)] +
               [(135, 64), (64,)] + _ENC28 + [(128, 256), (256,)] + _LSTM + [(32, 256), (256,), (32, 256)] + _LLC)
SEPMC_SHAPES = ([(1, 135), (1, 135), (135, 128), (128,)] + _ENC26 + [(64, 128), (128,), (29, 64), (64,), (64, 64), (64,), (64, 128), (128,), (384, 256), (256,)] +
                _LSTM + [(32, 1), (1,)] +
                [(135, 64), (64,)] + _ENC26 + [(29, 64), (64,), (64, 64), (64,), (192, 256), (256,)] + _LSTM + [(32, 1), (1,), (1, 1)] +
                [(135, 64), (64,)] + _ENC28 + [(128, 256), (256,)] + _LSTM + [(32, 256), (256,), (32, 256)] + _LLC)


def random_weights(strategic=False, seed=0):
    """Random weights of the shipped architecture (benchmarks, tests): fan-in scaled normals, positive running std."""
    rng = np.random.default_rng(seed)
    shapes = SEPMC_SHAPES if strategic else EPMC_SHAPES
    w = [(rng.standard_normal(s) / np.sqrt(max(1, int(np.prod(s[:-1]))))).astype(np.float32) for s in shapes]
    w[1] = np.abs(w[1]) + 0.2
    return w


# ---------------------------------------------------------------------------------------------------------------- device side
def hier_role_arrays(strategic, value_tower=False):
    """Index (in the shipped file's array list) of the array that plays each role of include/llq_policy.h; `value_tower`: the
    environmental level's value-tower table (LLQ_HIER_ROLES_VALUE entries) instead (the strategic level's training table is
    `strategic_train_role_arrays`)."""
    if value_tower:
        if strategic:
            raise ValueError("the value-tower table exists for the environmental level only (strategic level: strategic_train_role_arrays)")
        return list(range(2, 47))
    if not strategic:
        return [0, 1, 47, 48] + list(range(49, 77)) + [77, 78] + list(range(79, 88)) + [88, 89, 90] + list(range(91, 101))
    mlc = [0, 1, 97, 98] + list(range(99, 127)) + [127, 128] + list(range(129, 138)) + [138, 139, 140] + list(range(141, 151))
    hlc = [51, 52] + list(range(53, 79)) + [79, 80, 81, 82] + [83, 84] + list(range(85, 94)) + [94, 95]
    return mlc + hlc


def strategic_train_role_arrays():
    """The strategic level's training table (LLQ_HIER_ROLES_TRAIN_STRATEGIC entries, include/llq_policy.h): the value tower, arrays
    2-50 of strategic_level.model, then the heading logstd (array 96)."""
    return list(range(2, 51)) + [96]


def _policy_lib():
    import os
    from .policy import POLICY_LIB_PATH
    if not os.path.exists(POLICY_LIB_PATH):
        raise RuntimeError("%s is not built (python -c 'import __graft_entry__ as g; g.build()'); there is no CPU fallback" % POLICY_LIB_PATH)
    lib = C.CDLL(POLICY_LIB_PATH)
    lib.llq_hier_policy_last_error.restype = C.c_char_p
    return lib


def weight_blob(weights):
    """(blob, starts): the arrays concatenated as fp32, each starting on a 16-byte boundary (the kernel's float4 loads).  The one builder
    of the layout the device handles keep: a learner forms the blob it broadcasts to its actors with it (blob as a CUDA tensor goes to
    `set_weights` / `DeviceOpponentPool.set_model`)."""
    w = [np.ascontiguousarray(a, np.float32).reshape(-1) for a in weights]
    w = [np.concatenate([a, np.zeros((-a.size) % 4, np.float32)]) for a in w]
    starts = np.concatenate([[0], np.cumsum([a.size for a in w])]).astype(np.int64)
    return np.concatenate(w), starts


def _blob_and_tables(models, *roles):
    """(blob, tables): the arrays of all `models` in one fp32 blob, model after model (each laid out by `weight_blob`), and for each list
    of array indices in `roles` the int32 table of where those arrays start in the blob, model after model (the role tables of
    include/llq_policy.h)."""
    blobs, starts, base = [], [], 0
    for m in models:
        blob, s = weight_blob(m)
        blobs.append(blob)
        starts.append(s + base)
        base += blob.size
    blob = np.concatenate(blobs) if blobs else np.zeros(0, np.float32)
    return blob, [np.array([s[i] for s in starts for i in r], np.int32) for r in roles]


def pool_regions(offsets, n_models, n_weights):
    """[(lo, hi)] per model of a pool blob (include/llq_policy.h, llq_hier_policy_set_pool_model): model k's region runs from its smallest
    role offset to the next larger model start, or to the end of the blob; None when two models share arrays (two models starting at
    the same float, or one of model k's arrays starting outside its region).  `offsets`: the pool's [n_models * 101] role table."""
    off = np.asarray(offsets, np.int64).reshape(n_models, -1)
    lo = off.min(1)
    if len(set(lo.tolist())) < n_models:
        return None
    hi = [min([int(x) for x in lo if x > lo[k]], default=int(n_weights)) for k in range(n_models)]
    if any((off[k] >= hi[k]).any() for k in range(n_models)):
        return None
    return [(int(lo[k]), hi[k]) for k in range(n_models)]


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


class _HierHandle:
    """One handle of csrc/llq_policy_hier.cu (include/llq_policy.h): the library, its calls and `close`."""

    def __init__(self, create, *args):
        """`create`(*args, &handle): the library entry that makes the handle."""
        self.lib, self._h = _policy_lib(), None
        h = C.c_void_p()
        self._call(create, *args, C.byref(h))
        self._h = h

    def _call(self, entry, *args, error=RuntimeError):
        """The library's `entry`(*args); a non-zero return raises `error` with the library's last error."""
        if getattr(self.lib, entry)(*args):
            raise error("%s: %s" % (entry, self.lib.llq_hier_policy_last_error().decode()))

    def _refresh(self, entry, head, weights, n, shapes, what, stream):
        """`entry`(*head, weights, n, on_device, stream): the checks of a host list (the level's `shapes`) or a flat CUDA tensor of n floats,
        then the library call; a device source is kept from the allocator until the copy on `stream` has run."""
        if is_tensor(weights):
            check_device_blob(weights, n, self.device)
            ptr, on_device = weights.data_ptr(), 1
        else:
            check_arrays(weights, shapes, what)
            blob = weight_blob(weights)[0]
            if blob.size != n:
                raise ValueError("the blob of %s has %d floats, the handle expects %d" % (what, blob.size, n))
            ptr, on_device = blob.ctypes.data, 0
        self._call(entry, *head, C.c_void_p(ptr), C.c_int64(n), C.c_int32(on_device), C.c_void_p(stream or 0))
        if on_device:
            keep_for_stream(weights, stream, self.device)

    def set_weights(self, weights, stream=None):
        """The learner's new weights (include/llq_policy.h, llq_hier_policy_set_weights), asynchronous on `stream` (a cudaStream_t, None =
        the default stream): forwards queued there before see the old weights, forwards queued after it the new ones; the LSTM states
        are the caller's and stay.  `weights`: the level's arrays (102 / 152; the host list may be reused as soon as this returns), or a
        flat float32 CUDA tensor on the handle's device in the blob layout (`weight_blob(arrays)[0]`)."""
        self._refresh("llq_hier_policy_set_weights", (self._h,), weights, self.n_weights, SEPMC_SHAPES if self.strategic else EPMC_SHAPES,
                      "a strategic-level model" if self.strategic else "an environmental-level model", stream)

    def close(self):
        if self._h:
            self.lib.llq_hier_policy_destroy(self._h)
            self._h = None


class DeviceHierPolicy(_HierHandle):
    """The environmental- / strategic-level policy on the GPU (csrc/llq_policy_hier.cu through include/llq_policy.h): reads the engine's
    observation rows in place, keeps the LSTM states on the device, writes the actions the fused env step consumes.
    `train=True` (environmental level only): the training handle, stepped with `forward_rec` (sampled code, -log p, V; state rows of
    128 floats = code LSTM, then value LSTM); the strategic level's training handle is `DeviceSepmcTrainPolicy`."""

    def __init__(self, weights, device=0, train=False):
        assert len(weights) in (102, 152), "expected an environmental-level (102 arrays) or a strategic-level (152 arrays) model"
        self.strategic, self.train, self.device = len(weights) == 152, bool(train), int(device)
        if self.train:
            blob, (off, voff) = _blob_and_tables([weights], hier_role_arrays(self.strategic), hier_role_arrays(False, value_tower=True))
            super().__init__("llq_hier_policy_create_train", _vp(blob), C.c_int64(blob.size), _vp(off), C.c_int32(off.size), _vp(voff),
                             C.c_int32(voff.size), C.c_int32(int(self.strategic)), C.c_int32(device))      # a strategic handle is refused
        else:
            blob, (off,) = _blob_and_tables([weights], hier_role_arrays(self.strategic))
            super().__init__("llq_hier_policy_create", _vp(blob), C.c_int64(blob.size), _vp(off), C.c_int32(off.size),
                             C.c_int32(int(self.strategic)), C.c_int32(device))
        self.n_weights = blob.size
        self.state_dim = 128 if (self.strategic or self.train) else 64
        self.obs_dim = 965 if self.strategic else 916

    def forward(self, obs_ptr, obs_ld, n, done_ptr, state_ptr, act_ptr, codes_ptr=None, heading_ptr=None, stream=None):
        self._call("llq_hier_policy_forward", self._h, C.c_void_p(obs_ptr), C.c_int64(obs_ld), C.c_int32(n), C.c_void_p(done_ptr or 0),
                   C.c_void_p(state_ptr), C.c_void_p(act_ptr), C.c_void_p(codes_ptr or 0), C.c_void_p(heading_ptr or 0), C.c_void_p(stream or 0))

    def forward_rec(self, obs_ptr, obs_ld, n, done_ptr, state_ptr, act_ptr, codes_ptr, values_ptr, neglogp_ptr, out_ld, seed, counter, row_gid0=0,
                    stream=None):
        """Training step (include/llq_policy.h, llq_hier_policy_forward_rec): sampled code -> codes_ptr (int32), V / -log p of row i ->
        values_ptr / neglogp_ptr + i * out_ld floats; the Gumbel noise is keyed by (row_gid0 + i, counter) and `seed`."""
        self._call("llq_hier_policy_forward_rec", self._h, C.c_void_p(obs_ptr), C.c_int64(obs_ld), C.c_int32(n), C.c_void_p(done_ptr or 0),
                   C.c_void_p(state_ptr), C.c_void_p(act_ptr), C.c_void_p(codes_ptr or 0), C.c_void_p(values_ptr or 0), C.c_void_p(neglogp_ptr or 0),
                   C.c_int64(out_ld), C.c_uint64(seed), C.c_uint64(counter), C.c_int64(row_gid0), C.c_void_p(stream or 0))


class DeviceSepmcTrainPolicy(_HierHandle):
    """The strategic level's training handle on the GPU (include/llq_policy.h, llq_hier_policy_create_train_strategic): `forward_rec`
    samples the heading, writes it raw with its -log p and V, and runs the frozen code controller (argmax code) and decoder on the
    clipped heading.  State rows of 192 floats: heading LSTM, code LSTM, value LSTM ([c, h] each)."""

    def __init__(self, weights, device=0):
        assert len(weights) == 152, "expected a strategic-level model (152 arrays)"
        self.strategic, self.train, self.device = True, True, int(device)
        blob, (off, toff) = _blob_and_tables([weights], hier_role_arrays(True), strategic_train_role_arrays())
        super().__init__("llq_hier_policy_create_train_strategic", _vp(blob), C.c_int64(blob.size), _vp(off), C.c_int32(off.size), _vp(toff),
                         C.c_int32(toff.size), C.c_int32(device))
        self.n_weights = blob.size
        self.state_dim, self.obs_dim = 192, 965

    # the deterministic entry, which the library refuses for this handle: `forward` raises the library's RuntimeError (naming
    # llq_hier_policy_forward_rec_strategic, the entry to step with) rather than an AttributeError
    forward = DeviceHierPolicy.forward

    def forward_rec(self, obs_ptr, obs_ld, n, done_ptr, state_ptr, act_ptr, codes_ptr, heading_ptr, values_ptr, neglogp_ptr, out_ld, seed, counter,
                    row_gid0=0, stream=None):
        """Training step (include/llq_policy.h, llq_hier_policy_forward_rec_strategic): raw sampled heading / V / -log p of row i ->
        heading_ptr / values_ptr / neglogp_ptr + i * out_ld floats, argmax code -> codes_ptr (int32); the heading noise is keyed by
        (row_gid0 + i, counter) and `seed`."""
        self._call("llq_hier_policy_forward_rec_strategic", self._h, C.c_void_p(obs_ptr), C.c_int64(obs_ld), C.c_int32(n), C.c_void_p(done_ptr or 0),
                   C.c_void_p(state_ptr), C.c_void_p(act_ptr), C.c_void_p(codes_ptr or 0), C.c_void_p(heading_ptr or 0), C.c_void_p(values_ptr or 0),
                   C.c_void_p(neglogp_ptr or 0), C.c_int64(out_ld), C.c_uint64(seed), C.c_uint64(counter), C.c_int64(row_gid0), C.c_void_p(stream or 0))


class DeviceOpponentPool(_HierHandle):
    """K frozen strategic-level models on the GPU in one handle (include/llq_policy.h, llq_hier_policy_create_pool): `forward` draws a
    new model for every row whose done flag is set, from the probabilities of `set_probs` (uniform until then), and runs every row's
    deterministic forward with its own model in one launch.  `models`: a list of 1 .. 64 strategic-level models (152 arrays each);
    `max_rows` bounds the rows of every forward.  Single-owner: the handle holds one workspace, so one stream at a time."""

    def __init__(self, models, device=0, *, max_rows, probs=None):
        assert all(len(m) == 152 for m in models), "expected strategic-level models (152 arrays)"
        self.strategic, self.train, self.device = True, False, int(device)
        self.n_models, self.max_rows = len(models), int(max_rows)
        self.state_dim, self.obs_dim = 128, 965
        blob, (off,) = _blob_and_tables(models, hier_role_arrays(True))
        super().__init__("llq_hier_policy_create_pool", _vp(blob), C.c_int64(blob.size), _vp(off), C.c_int32(self.n_models), C.c_int32(self.max_rows),
                         C.c_int32(device))
        self.n_weights, self.regions = blob.size, pool_regions(off, self.n_models, blob.size)
        if probs is not None:
            self.set_probs(probs)

    def set_weights(self, weights, stream=None):
        raise ValueError("a pool replaces one model at a time: set_model(k, weights)")

    def set_model(self, k, weights, stream=None):
        """Replaces model k (include/llq_policy.h, llq_hier_policy_set_pool_model), asynchronous on `stream` as `set_weights` is; the
        number of models stays.  `weights`: a strategic-level model (152 arrays), or a flat float32 CUDA tensor on the handle's device
        holding `weight_blob(arrays)[0]`.  Pairs whose current game is against model k continue it with the new weights and the state
        they carry; a model with probability 0 can be filled here and given a probability later (`set_probs`)."""
        if not 0 <= int(k) < self.n_models:
            raise ValueError("model index %s outside [0, %d)" % (k, self.n_models))
        if self.regions is None:
            raise ValueError("the pool's models share arrays: no model has a region of its own")
        lo, hi = self.regions[int(k)]
        self._refresh("llq_hier_policy_set_pool_model", (self._h, C.c_int32(int(k))), weights, hi - lo, SEPMC_SHAPES, "a strategic-level model",
                      stream)

    def set_probs(self, probs):
        """Draw probabilities of the next forwards: one finite entry >= 0 per model, positive sum (they need not sum to 1)."""
        p = np.ascontiguousarray(probs, np.float64).reshape(-1)
        self._call("llq_hier_policy_set_pool_probs", self._h, _vp(p), C.c_int32(p.size), error=ValueError)

    def forward(self, obs_ptr, obs_ld, n, done_ptr, state_ptr, act_ptr, codes_ptr, heading_ptr, model_ptr, model_rec_ptr, rec_ld, seed, counter,
                row_gid0=0, stream=None):
        """One step (include/llq_policy.h, llq_hier_policy_forward_pool): rows with done set draw a model into model_ptr (int32[n]), keyed
        by (row_gid0 + i, counter) and `seed`; model_rec_ptr + i * rec_ld floats (nullable) records every row's model."""
        self._call("llq_hier_policy_forward_pool", self._h, C.c_void_p(obs_ptr), C.c_int64(obs_ld), C.c_int32(n), C.c_void_p(done_ptr or 0),
                   C.c_void_p(state_ptr), C.c_void_p(act_ptr), C.c_void_p(codes_ptr or 0), C.c_void_p(heading_ptr or 0), C.c_void_p(model_ptr),
                   C.c_void_p(model_rec_ptr or 0), C.c_int64(rec_ld), C.c_uint64(seed), C.c_uint64(counter), C.c_int64(row_gid0),
                   C.c_void_p(stream or 0))
