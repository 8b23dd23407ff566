"""NumPy models of MAPPO's actor in the in-kernel rollout (env.rollout_policy with LayerNorm policies,
mpe_rollout_policy_mappo): the float64 evaluation of the folded network with the kernel's recipe -- statistics of every
LayerNorm, then TF32 (cvt.rna) rounding of every GEMM operand (the normalised x0, x1, x2 and the folded weights), fp32
biases -- the float64 evaluation of the user's unfolded module, seeded MAPPO actors, and the accounting for every pick
or log-probability that differs from the model: TF32 rounding flips of the normalised operands, or the Gumbel gap."""
import itertools

import numpy as np

from mlp_categorical_helpers import LOGP_ATOL, _row_ok, categorical_pick, log_softmax_at
from mlp_helpers import flip_candidates, tf32_accumulation_bound, tf32_rna

H = 64
FEATURE_NORM, TANH = 1, 2          # net_flags
# flip combinations tried per row.  More than mlp_helpers' 2^6: a row has up to three layers of ambiguous operands here
# (the input LayerNorm's too), and a LayerNorm couples all units of a row through its statistics.  At 2^8, 10 of the 68
# replay cases each left one row unexplained after every combination tried (rows whose explanation needs two or three
# flips among a dozen ambiguous groups)
MAPPO_MAX_COMBOS = 2 ** 12
U = 2.0 ** -24


def layer_norm(x, eps):
    """parameter-free LayerNorm over the last axis, float64, two-pass as torch"""
    mu = x.mean(-1, keepdims=True)
    var = ((x - mu) ** 2).mean(-1, keepdims=True)
    return (x - mu) / np.sqrt(var + eps)


def activation(x, tanh):
    return np.tanh(x) if tanh else np.maximum(x, 0.0)


def norm_error_bound(a, ea, eps):
    """per-element bound on |fp32 LayerNorm(a') - float64 LayerNorm(a)| where the kernel's input a' is within ea of a
    (elementwise, [m, K]): the error of a and of the mean carried through 1 / sigma, and the fp32 sums of K terms
    (sequential or a shuffle tree), the rsqrtf and the products, generously as (K + 8) u times |x| and mean |a| / sigma"""
    K = a.shape[-1]
    sigma = np.sqrt(((a - a.mean(-1, keepdims=True)) ** 2).mean(-1, keepdims=True) + eps)
    x = (a - a.mean(-1, keepdims=True)) / sigma
    return (ea + ea.mean(-1, keepdims=True)) / sigma + (K + 8) * U * (np.abs(x) + np.abs(a).mean(-1, keepdims=True) / sigma)


def flip_choices(x, bound):
    """(x rounded to TF32 as the model does, the other TF32 value a value within `bound` of x may round to -- NaN where
    the element is not ambiguous)"""
    f32 = np.float32
    r = tf32_rna(x.astype(f32)).astype(np.float64)
    lo = tf32_rna((x - bound).astype(f32)).astype(np.float64)
    hi = tf32_rna((x + bound).astype(f32)).astype(np.float64)
    return r, np.where(lo != r, lo, np.where(hi != r, hi, np.nan))


class MappoModel:
    """the kernel's recipe in float64 for one agent: params = the folded (W1, b1, W2, b2, W3, b3) as float32, i.e. what
    the kernel is given; net = (net_flags, eps)"""

    def __init__(self, params, net):
        f64 = np.float64
        W1, b1, W2, b2, W3, b3 = [np.asarray(p, dtype=np.float32) for p in params]
        self.t = [tf32_rna(W).astype(f64) for W in (W1, W2, W3)]
        self.b = [np.asarray(b, f64) for b in (b1, b2, b3)]
        self.flags, self.eps = int(net[0]), float(net[1])
        self.tanh = bool(self.flags & TANH)

    def input(self, obs):
        """(normalised input x0 before its rounding, its error bound or None)"""
        o = np.asarray(obs, np.float64)
        if not self.flags & FEATURE_NORM:
            return o, None
        return layer_norm(o, self.eps), norm_error_bound(o, np.zeros_like(o), self.eps)

    def hidden(self, x_rounded, layer):
        """(normalised act(x . W^T + b) before its rounding, its error bound)"""
        t, b = self.t[layer], self.b[layer]
        p = x_rounded @ t.T + b
        a = activation(p, self.tanh)
        ea = tf32_accumulation_bound(x_rounded, t, b) + (2 * U * np.abs(a) if self.tanh else 0.0)
        return layer_norm(a, self.eps), norm_error_bound(a, ea, self.eps)

    def logits(self, x2_rounded):
        return x2_rounded @ self.t[2].T + self.b[2]

    def __call__(self, obs):
        rnd = lambda v: tf32_rna(v.astype(np.float32)).astype(np.float64)   # noqa: E731
        x0 = rnd(self.input(obs)[0])
        x1 = rnd(self.hidden(x0, 0)[0])
        x2 = rnd(self.hidden(x1, 1)[0])
        return self.logits(x2)


def module_logits(module, obs):
    """the user's unfolded nn.Sequential in float64 on the CPU"""
    import copy

    import torch
    m = copy.deepcopy(module).to(device="cpu", dtype=torch.float64)
    with torch.no_grad():
        return m(torch.as_tensor(np.asarray(obs, np.float64))).numpy()


def ambiguous_groups(values, alt):
    """the ambiguous elements of one row (alt not NaN), grouped by equal value: [(index, ...), ...]"""
    groups = {}
    for j in np.where(~np.isnan(alt))[0]:
        groups.setdefault(float(values[j]), []).append(int(j))
    return [tuple(g) for g in groups.values()]


def next_layer(model, layer_index):
    """flip_candidates' layer after a rounded row: (rounded values, alternatives, ambiguous groups) of hidden layer
    `layer_index`"""
    def of(prev):
        v, e = model.hidden(prev[None], layer_index)
        r, alt = flip_choices(v[0], e[0])
        return r, alt, ambiguous_groups(v[0], alt)
    return of


def explain_mappo_mismatches(k, logp, obs, model, segments, noise=0.0):
    """Assert that every row whose pick k [n, n_sub] differs from the arg-max of the float64 model (+ noise), or whose
    log-probability logp [n] is more than LOGP_ATOL from the model's log_softmax at k, is explained by
      - a combination of TF32 rounding flips of the normalised operands x0 (with the input LayerNorm), x1 and x2: an
        operand is ambiguous when the kernel's fp32 value may lie on the other side of a TF32 rounding boundary
        (norm_error_bound), and a flip of x0 or x1 is carried into the next layer's values and ambiguity; or
      - in a sub-space whose pick differs, a float64 gap between the two perturbed logits within GUMBEL_GAP.
    Operands of one row with the same float64 value -- after ReLU every inactive unit of a row normalises to the same
    -mu / sigma -- are the same fp32 value in the kernel too, so they flip together: a flip is one such group.
    Flip sets are tried in order of their size, earlier layers first, at most MAPPO_MAX_COMBOS per row.
    Returns (rows explained by a flip, rows explained by the Gumbel gap)."""
    n = k.shape[0]
    noise = np.broadcast_to(np.asarray(noise, np.float64), (n, model.t[2].shape[0]))
    x0v, e0 = model.input(obs)
    x0 = tf32_rna(x0v.astype(np.float32)).astype(np.float64)
    x1v, _ = model.hidden(x0, 0)
    x1 = tf32_rna(x1v.astype(np.float32)).astype(np.float64)
    x2v, _ = model.hidden(x1, 1)
    x2 = tf32_rna(x2v.astype(np.float32)).astype(np.float64)
    z = model.logits(x2)
    bad = np.where((categorical_pick(z + noise, segments) != k).any(-1) |
                   (np.abs(log_softmax_at(z, k, segments) - logp) > LOGP_ATOL))[0]
    flips, gaps, unexplained = 0, 0, []
    for w in bad:
        lp = float(logp[w])
        ok, gap = _row_ok(z[w], noise[w], k[w], lp, segments)
        if ok:
            gaps += 1
            continue
        if e0 is not None:
            _, alt0 = flip_choices(x0v[w], e0[w])
        else:
            alt0 = np.full(x0v.shape[1], np.nan)
        first = (x0[w], alt0, ambiguous_groups(x0v[w], alt0))
        tried, ok = 0, False
        for g in itertools.islice(flip_candidates(first, [next_layer(model, 0), next_layer(model, 1)]),
                                  MAPPO_MAX_COMBOS):
            tried += 1
            ok, _ = _row_ok(model.logits(g), noise[w], k[w], lp, segments)
            if ok:
                break
        if ok:
            flips += 1
        else:
            unexplained.append((int(w), k[w].tolist(), categorical_pick((z + noise)[w:w + 1], segments)[0].tolist(),
                                lp, float(log_softmax_at(z[w:w + 1], k[w:w + 1], segments)[0]), tried))
    assert not unexplained, ("%d of %d rows are neither TF32 rounding flips of the normalised operands nor within the "
                             "Gumbel gap (row, pick, model pick, logp, model logp, combinations tried): %s"
                             % (len(unexplained), bad.size, unexplained[:8]))
    return flips, gaps


def make_mappo_actors(obs_dims, act_dims, tanh, feature_norm, seed=3, eps=1e-5, device="cuda", hidden=H):
    """seeded MAPPO actors (nn.Sequential) with non-trivial LayerNorm affines; every third Linear weight on a TF32
    rounding tie, so that a rounding mode other than ties-away shows"""
    import torch
    from mlp_helpers import tf32_tie
    nn = torch.nn
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float32)   # noqa: E731
    Act = nn.Tanh if tanh else nn.ReLU
    mods = []
    for od, ad in zip(obs_dims, act_dims):
        layers = ([nn.LayerNorm(od, eps=eps)] if feature_norm else []) + [
            nn.Linear(od, hidden), Act(), nn.LayerNorm(hidden, eps=eps), nn.Linear(hidden, hidden), Act(),
            nn.LayerNorm(hidden, eps=eps), nn.Linear(hidden, ad)]
        m = nn.Sequential(*layers)
        with torch.no_grad():
            for layer in m:
                if isinstance(layer, nn.Linear):
                    layer.weight.copy_(torch.as_tensor(tf32_tie((r(*layer.weight.shape) * 1.5 / layer.in_features ** 0.5)
                                                                .numpy(), 3)))
                    layer.bias.copy_(r(layer.out_features) * 0.3)
                elif isinstance(layer, nn.LayerNorm):
                    layer.weight.copy_(1.0 + 0.3 * r(*layer.weight.shape))
                    layer.bias.copy_(0.2 * r(*layer.bias.shape))
        mods.append(m.to(device))
    return mods
