"""NumPy models of MAPPO's recurrent actor in the in-kernel rollout (env.rollout_policy with a (base, gru, norm, head)
tuple, mpe_rollout_policy_gru): the float64 evaluation of the folded network with the kernel's recipe -- TF32 (cvt.rna)
rounding of the normalised base output x, of h as the A operand of W_hh, of LN(h') and of every weight, with the
rounding switchable off -- the float64 evaluation of the user's unfolded modules, a written bound on the kernel's h'
given the same (o_t, h_t), seeded actors, and the accounting for every pick or log-probability that differs from the
model evaluated on the kernel's own h'."""
import itertools

import numpy as np

from mappo_helpers import (FEATURE_NORM, MAPPO_MAX_COMBOS, TANH, U, activation, ambiguous_groups, flip_choices,
                           layer_norm, norm_error_bound)
from mlp_categorical_helpers import LOGP_ATOL, _row_ok, categorical_pick, log_softmax_at
from mlp_helpers import flip_candidates, tf32_accumulation_bound, tf32_rna

H = 64
TF32_ULP = 2.0 ** -10      # one TF32 ulp of a value v is at most 2^-10 |v|: what a rounding flip moves an operand by


def sigmoid(v):
    return 1.0 / (1.0 + np.exp(-v))


class RecurrentModel:
    """The kernel's recipe in float64: params = rmappo_actor_params' folded (W1, b1, W2, b2, W_ih, b_ih, W_hh, b_hh,
    W3, b3), net = (net_flags, eps).  tf32=True models what the kernel is given and computes: the parameters cast to
    float32, the weights and the GEMMs' A operands rounded to TF32.  tf32=False keeps the float64 parameters and never
    rounds: the folded network exactly."""

    def __init__(self, params, net, tf32=True):
        f64 = np.float64
        ps = [np.asarray(p, np.float32 if tf32 else f64).astype(f64) for p in params]
        self.rnd = (lambda v: tf32_rna(np.asarray(v).astype(np.float32)).astype(f64)) if tf32 else (lambda v: v)
        self.W = [self.rnd(ps[j]) for j in (0, 2, 4, 6, 8)]          # W1, W2, W_ih, W_hh, W3
        self.b = [ps[j] for j in (1, 3, 5, 7, 9)]
        self.flags, self.eps = int(net[0]), float(net[1])
        self.tanh = bool(self.flags & TANH)

    def base(self, obs):
        """x: the normalised base output, rounded"""
        x = np.asarray(obs, np.float64)
        if self.flags & FEATURE_NORM:
            x = layer_norm(x, self.eps)
        x = self.rnd(x)
        for layer in (0, 1):
            x = self.rnd(layer_norm(activation(x @ self.W[layer].T + self.b[layer], self.tanh), self.eps))
        return x

    def gates(self, x, h):
        """(r, z, W_in x + b_in, W_hn h + b_hn) for the rounded x and the state h"""
        hr = self.rnd(np.asarray(h, np.float64))
        gi = x @ self.W[2].T + self.b[2]
        gh = hr @ self.W[3].T + self.b[3]
        return sigmoid(gi[:, :H] + gh[:, :H]), sigmoid(gi[:, H:2 * H] + gh[:, H:2 * H]), gi[:, 2 * H:], gh[:, 2 * H:]

    def gru(self, x, h):
        r, z, ni, nh = self.gates(x, h)
        return (1.0 - z) * np.tanh(ni + r * nh) + z * np.asarray(h, np.float64)

    def logits(self, hn):
        return self.rnd(layer_norm(np.asarray(hn, np.float64), self.eps)) @ self.W[4].T + self.b[4]

    def step(self, obs, h):
        """(logits, h') of one step"""
        hn = self.gru(self.base(obs), h)
        return self.logits(hn), hn

    def h_bound(self, obs, h, flips):
        """Per-element bound on |kernel h' - model h'| for the same (obs, h).  The kernel's normalised operands are fp32
        values within norm_error_bound of the model's float64 ones; rounded to TF32 they are either the model's
        (flips=False) or one TF32 ulp away (flips=True: every operand of the input, both hidden layers and x may flip,
        and each flip is carried through the next layer's GEMM and LayerNorm).  Then the fp32 tensor-core sums of the
        gates (tf32_accumulation_bound over the 128 terms of r and z, 64 of each n part), the operand error of x through
        |W_ih|, expf / tanhf / the division to a few ulp, sigmoid' <= 1/4 and tanh' <= 1, and
        h' = (1 - z) n + z h: |dh'| <= |dz| |n - h| + (1 - z) |dn| + 4u (|n| + |h|)."""
        f64 = np.float64
        o = np.asarray(obs, f64)
        d = np.zeros_like(o)
        x = o
        if self.flags & FEATURE_NORM:
            v = layer_norm(o, self.eps)
            if flips:
                d = TF32_ULP * (np.abs(v) + norm_error_bound(o, np.zeros_like(o), self.eps))
            x = v
        x = self.rnd(x)
        for layer in (0, 1):
            W, b = self.W[layer], self.b[layer]
            a = activation(x @ W.T + b, self.tanh)
            ea = tf32_accumulation_bound(x, W, b) + d @ np.abs(W).T + (2 * U * np.abs(a) if self.tanh else 0.0)
            v = layer_norm(a, self.eps)
            d = TF32_ULP * (np.abs(v) + norm_error_bound(a, ea, self.eps)) if flips else np.zeros_like(v)
            x = self.rnd(v)
        hh = np.asarray(h, f64)
        hr = self.rnd(hh)
        Wi, Wh, bi, bh = self.W[2], self.W[3], self.b[2], self.b[3]
        err = []
        for g in (slice(0, H), slice(H, 2 * H)):               # r and z: both GEMMs and both biases in one sum
            err.append(tf32_accumulation_bound(np.hstack([x, hr]), np.hstack([Wi[g], Wh[g]]), bi[g] + bh[g]) +
                       d @ np.abs(Wi[g]).T)
        g = slice(2 * H, 3 * H)
        e_ni = tf32_accumulation_bound(x, Wi[g], bi[g]) + d @ np.abs(Wi[g]).T
        e_nh = tf32_accumulation_bound(hr, Wh[g], bh[g])
        r, z, ni, nh = self.gates(x, hh)
        n = np.tanh(ni + r * nh)
        dr, dz = err[0] / 4 + 4 * U, err[1] / 4 + 4 * U
        darg = e_ni + r * e_nh + np.abs(nh) * dr + 2 * U * (np.abs(ni) + np.abs(r * nh))
        dn = darg + 4 * U
        return dz * np.abs(n - hh) + (1.0 - z) * dn + 4 * U * (np.abs(n) + np.abs(hh))


def module_step(actor, obs, h):
    """the user's unfolded (base, gru, norm, head) in float64 on the CPU: (logits, h')"""
    import copy

    import torch
    base, gru, norm, head = [copy.deepcopy(m).to(device="cpu", dtype=torch.float64) for m in actor]
    with torch.no_grad():
        x = base(torch.as_tensor(np.asarray(obs, np.float64)))
        out, hn = gru(x[None], torch.as_tensor(np.asarray(h, np.float64))[None])
        return head(norm(out[0])).numpy(), hn[0].numpy()


def explain_head_mismatches(k, logp, hn, model, segments, noise=0.0):
    """Assert that every row whose pick k [n, n_sub] differs from the arg-max of model.logits(hn) (+ noise), hn the
    kernel's own h', or whose log-probability differs by more than LOGP_ATOL, is explained by TF32 rounding flips of
    LN(h') (the kernel's fp32 LayerNorm within norm_error_bound of the float64 one; equal values flip together) or by
    the Gumbel gap.  Returns (rows explained by a flip, rows explained by the Gumbel gap)."""
    n = k.shape[0]
    noise = np.broadcast_to(np.asarray(noise, np.float64), (n, model.W[4].shape[0]))
    hn = np.asarray(hn, np.float64)
    v = layer_norm(hn, model.eps)
    e = norm_error_bound(hn, np.zeros_like(hn), model.eps)
    z = model.logits(hn)
    bad = np.where((categorical_pick(z + noise, segments) != k).any(-1) |
                   (np.abs(log_softmax_at(z, k, segments) - logp) > LOGP_ATOL))[0]
    flips, gaps, unexplained = 0, 0, []
    for w in bad:
        lp = float(logp[w])
        ok, _ = _row_ok(z[w], noise[w], k[w], lp, segments)
        if ok:
            gaps += 1
            continue
        r, alt = flip_choices(v[w], e[w])
        for g in itertools.islice(flip_candidates((r, alt, ambiguous_groups(v[w], alt)), []), MAPPO_MAX_COMBOS):
            ok, _ = _row_ok(g @ model.W[4].T + model.b[4], noise[w], k[w], lp, segments)
            if ok:
                break
        if ok:
            flips += 1
        else:
            unexplained.append((int(w), k[w].tolist(), categorical_pick((z + noise)[w:w + 1], segments)[0].tolist(), lp,
                                float(log_softmax_at(z[w:w + 1], k[w:w + 1], segments)[0])))
    assert not unexplained, ("%d of %d rows are neither TF32 rounding flips of LN(h') nor within the Gumbel gap (row, "
                             "pick, model pick, logp, model logp): %s" % (len(unexplained), bad.size, unexplained[:8]))
    return flips, gaps


def make_rmappo_actor(obs_dim, act_dim, tanh, feature_norm, seed=3, eps=1e-5, device="cuda"):
    """one seeded (base, gru, norm, head) with non-trivial LayerNorm affines and GRU weights at torch's default
    scale"""
    import torch
    nn = torch.nn
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float32)   # noqa: E731
    Act = nn.Tanh if tanh else nn.ReLU
    base = nn.Sequential(*(([nn.LayerNorm(obs_dim, eps=eps)] if feature_norm else []) + [
        nn.Linear(obs_dim, H), Act(), nn.LayerNorm(H, eps=eps), nn.Linear(H, H), Act(), nn.LayerNorm(H, eps=eps)]))
    gru, norm, head = nn.GRU(H, H), nn.LayerNorm(H, eps=eps), nn.Linear(H, act_dim)
    with torch.no_grad():
        for m in list(base) + [norm, head]:
            if isinstance(m, nn.Linear):
                m.weight.copy_(r(*m.weight.shape) * 1.5 / m.in_features ** 0.5)
                m.bias.copy_(r(m.out_features) * 0.3)
            elif isinstance(m, nn.LayerNorm):
                m.weight.copy_(1.0 + 0.3 * r(*m.weight.shape))
                m.bias.copy_(0.2 * r(*m.bias.shape))
        for p in gru.parameters():
            p.copy_(r(*p.shape) * 1.5 / H ** 0.5)
    return tuple(m.to(device) for m in (base, gru, norm, head))
