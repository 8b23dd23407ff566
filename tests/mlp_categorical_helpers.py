"""NumPy models of the categorical form of the two-hidden-layer in-kernel actor (env.rollout_policy(...,
action_mode="categorical")): the arg-max per action sub-space, its log-probability, the one-hot replay of the index
records, and the accounting for every pick or log-probability that differs from the float64 model of the TF32 actor.
The building blocks (TF32 rounding, the accumulation bound, the flip choices) are the ones of mlp_helpers."""
import itertools

import numpy as np

from mlp_helpers import (TF32_MAX_COMBOS, flip_candidates, relu_layer, relu_next_layer, tf32_accumulation_bound,
                         tf32_flip_choices, tf32_rna)

# the fp32 error of the kernel's Gumbel term logf(-logf(u)) next to float64 -log(-log u): a few ulps of values below 17
GUMBEL_GAP = 1e-5
LOGP_ATOL = 1e-5


def bounds(segments):
    """(start, end) of every sub-space"""
    b = np.cumsum([0] + list(segments))
    return list(zip(b[:-1], b[1:]))


def categorical_pick(z, segments):
    """int [n, n_sub]: the arg-max of every sub-space, the lowest index winning ties (np.argmax)"""
    return np.stack([np.argmax(z[:, a:b], -1) for a, b in bounds(segments)], -1).astype(np.int32)


def log_softmax_at(z, k, segments):
    """float64 [n]: sum over sub-spaces, in order, of log_softmax(z[:, segment])[k]"""
    out = np.zeros(z.shape[0])
    for s, (a, b) in enumerate(bounds(segments)):
        seg = z[:, a:b]
        m = seg.max(-1, keepdims=True)
        lsm = seg - m - np.log(np.exp(seg - m).sum(-1, keepdims=True))
        out += np.take_along_axis(lsm, k[:, s:s + 1].astype(np.int64), 1)[:, 0]
    return out


def one_hot(k, segments):
    """float32 [n, act_dim]: the action vector the kernel applies for the indices k [n, n_sub]"""
    out = np.zeros((k.shape[0], sum(segments)), np.float32)
    for s, (a, b) in enumerate(bounds(segments)):
        out[np.arange(k.shape[0]), a + k[:, s]] = 1.0
    return out


def one_hot_torch(k, segments):
    """the same on the device: int32 [n, n_sub] -> float32 [n, act_dim]"""
    import torch
    return torch.cat([torch.nn.functional.one_hot(k[:, s].long(), b - a).float()
                      for s, (a, b) in enumerate(bounds(segments))], -1)


def _row_ok(g, noise, k, logp, segments):
    """do the logits g (one row) explain the pick k and the log-probability logp?  Returns (ok, needed the Gumbel gap)"""
    zp = g + noise
    gap_used = False
    for s, (a, b) in enumerate(bounds(segments)):
        j = a + int(np.argmax(zp[a:b]))
        if j != a + int(k[s]):
            if zp[j] - zp[a + int(k[s])] > GUMBEL_GAP:
                return False, False
            gap_used = True
    if logp is not None and abs(log_softmax_at(g[None], k[None], segments)[0] - logp) > LOGP_ATOL:
        return False, False
    return True, gap_used


def split_pick_noise(z_model, z_kernel):
    """Noise for one row of one sub-space under which the model's logits z_model and the kernel's z_kernel pick
    different entries: the pair of entries that z_kernel - z_model moves furthest apart, D, is set D / 2 apart, and every
    other entry far below.  Returns (noise, the kernel's pick, D / 2)."""
    d = z_kernel - z_model
    a, b = int(np.argmin(d)), int(np.argmax(d))
    half = (d[b] - d[a]) / 2
    noise = np.full(z_model.shape, -50.0)
    noise[a] = 0.0
    noise[b] = z_model[a] - z_model[b] - half
    return noise, b, half


def explain_categorical_mismatches(k, logp, obs, params, segments, noise=0.0):
    """Assert that every row whose pick k [n, n_sub] differs from the arg-max of the float64 TF32 model (+ noise), or
    whose log-probability logp [n] (None: not checked) is more than LOGP_ATOL from log_softmax of that model at k, is
    explained by one of
      - a TF32 rounding-flip combination (mlp_helpers' accounting: the same ambiguous units, bound, order and
        combination limit) under which the pick is the arg-max and the log-probability is within LOGP_ATOL;
      - in a sub-space whose pick differs, a float64 gap between the two perturbed logits within GUMBEL_GAP.
    Returns (rows explained by a flip, rows explained by the Gumbel gap)."""
    f64 = np.float64
    W1, b1, W2, b2, W3, b3 = [np.asarray(p, dtype=np.float32) for p in params]
    t1, t2, t3 = (tf32_rna(W).astype(f64) for W in (W1, W2, W3))
    b1, b2, b3 = (np.asarray(b, f64) for b in (b1, b2, b3))
    n = k.shape[0]
    noise = np.broadcast_to(np.asarray(noise, f64), (n, W3.shape[0]))
    x0 = tf32_rna(obs).astype(f64)
    p1 = x0 @ t1.T + b1
    h1 = tf32_rna(np.maximum(p1, 0.0).astype(np.float32)).astype(f64)
    h2 = tf32_rna(np.maximum(h1 @ t2.T + b2, 0.0).astype(np.float32)).astype(f64)
    z = h2 @ t3.T + b3
    bad = np.where((categorical_pick(z + noise, segments) != k).any(-1) |
                   (np.abs(log_softmax_at(z, k, segments) - logp) > LOGP_ATOL if logp is not None else False))[0]
    flips, gaps, unexplained = 0, 0, []
    if bad.size == 0:
        return 0, 0
    _, alt1 = tf32_flip_choices(p1[bad], tf32_accumulation_bound(x0[bad], t1, b1))
    for r, w in enumerate(bad):
        lp = None if logp is None else float(logp[w])
        ok, gap = _row_ok(z[w], noise[w], k[w], lp, segments)
        if ok:
            gaps += 1
            continue
        tried = 0
        for g in itertools.islice(flip_candidates(relu_layer(h1[w], alt1[r]), [relu_next_layer(t2, b2)]),
                                  TF32_MAX_COMBOS):
            tried += 1
            ok, _ = _row_ok(g @ t3.T + b3, noise[w], k[w], lp, segments)
            if ok:
                break
        if ok:
            flips += 1
        else:
            unexplained.append((int(w), k[w].tolist(), categorical_pick((z + noise)[w:w + 1], segments)[0].tolist(),
                                lp, float(log_softmax_at(z[w:w + 1], k[w:w + 1], segments)[0]), tried))
    assert not unexplained, ("%d of %d rows are neither TF32 rounding flips nor within the Gumbel gap (row, pick, "
                             "model pick, logp, model logp, combinations tried): %s"
                             % (len(unexplained), bad.size, unexplained[:8]))
    return flips, gaps
