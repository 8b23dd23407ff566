"""NumPy models of the two-hidden-layer in-kernel actor for agents whose action vector has more than the 5 movement
entries (speakers, immovable agents): the Gumbel noise stream of act_dim logits, one softmax per action sub-space, the
TF32 accounting with that softmax, and the block-size cap of those programs.  The building blocks (TF32 rounding,
Philox, the accumulation bound and the flip choices) are the ones of mlp_helpers."""
import itertools

import numpy as np

from helpers import mlp_block_cap as _mlp_block_cap
from mlp_helpers import (EXPLORE_TAG, TF32_MAX_COMBOS, philox4x32_10, softmax, tf32_accumulation_bound,
                         tf32_flip_choices, tf32_rna, uniform_from_bits)


def gumbel_noise(seed, epoch, world_index, t, agent, n_agents, n_logits=5, stride=2):
    """-log(-log u) of the `n_logits` logits of `agent` at step `t` for the given global world indices, float64.  Logit
    k uses word k mod 4 of Philox block b = k div 4, counter word 3 = EXPLORE_TAG | ((t * n_agents + agent) * stride + b);
    stride is 2 when every action vector of the scenario has at most 8 entries, else 4.  The defaults are the stream of
    mlp_helpers.gumbel_noise."""
    gw = np.asarray(world_index, dtype=np.uint64)
    key = (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    base = EXPLORE_TAG | ((t * n_agents + agent) * stride)
    words = []
    for b in range((n_logits + 3) // 4):
        ctr = np.stack([gw & np.uint64(0xFFFFFFFF), gw >> np.uint64(32), np.full_like(gw, epoch & 0xFFFFFFFF),
                        np.full_like(gw, base | b)], -1)
        words.append(philox4x32_10(ctr, key))
    bits = np.concatenate(words, 1)[:, :n_logits]
    return -np.log(-np.log(uniform_from_bits(bits).astype(np.float64)))


def segment_softmax(z, segments=None):
    """one softmax per action sub-space: `segments` lists their widths in order (None: one softmax over the row)"""
    if segments is None:
        return softmax(z)
    assert sum(segments) == z.shape[-1], (segments, z.shape)
    bounds = np.cumsum([0] + list(segments))
    return np.concatenate([softmax(z[..., a:b]) for a, b in zip(bounds[:-1], bounds[1:])], -1)


def mlp_block_cap(H, n_agents, max_act_dim=5):
    """mlp_block_warps in csrc/mpe_kernels.cu: helpers.mlp_block_cap, plus 12 warps at H = 64 for a program with an
    action vector longer than 8 entries (simple_reference: 15)"""
    return 12 if (H == 64 and max_act_dim > 8) else _mlp_block_cap(H, n_agents)


def explain_tf32_mismatches(actions, obs, params, noise=0.0, atol=1e-5, segments=None):
    """mlp_helpers.explain_tf32_mismatches with the actions [n, act_dim] taken as one softmax per action sub-space
    (`segments`: their widths, e.g. [5, 10]; None: one softmax over the row).  Every row that differs from the TF32
    model by more than atol must be brought within atol by rounding some combination of its ambiguous h1 / h2 units the
    other way -- the same units, bound, order and combination limit as mlp_helpers.  Returns the number of explained
    rows."""
    f64 = np.float64
    W1, b1, W2, b2, W3, b3 = [np.asarray(p, dtype=np.float32) for p in params]
    H = W1.shape[0]
    t1, t2, t3 = (tf32_rna(W).astype(f64) for W in (W1, W2, W3))
    b1, b2, b3 = (np.asarray(b, f64) for b in (b1, b2, b3))
    got = np.asarray(actions, f64)
    noise = np.broadcast_to(np.asarray(noise, f64), got.shape)
    x0 = tf32_rna(obs).astype(f64)
    p1 = x0 @ t1.T + b1
    h1 = tf32_rna(np.maximum(p1, 0.0).astype(np.float32)).astype(f64)
    h2 = tf32_rna(np.maximum(h1 @ t2.T + b2, 0.0).astype(np.float32)).astype(f64)
    want = segment_softmax(h2 @ t3.T + b3 + noise, segments)
    bad = np.where((np.abs(got - want) > atol).any(-1))[0]
    if bad.size == 0:
        return 0
    _, alt1 = tf32_flip_choices(p1[bad], tf32_accumulation_bound(x0[bad], t1, b1))
    unexplained = []
    for r, w in enumerate(bad):
        amb1 = list(np.where(~np.isnan(alt1[r]))[0])
        h2_of = {}                                   # h1 flip set -> (h2 as the model rounds it, alternatives, ambiguous)

        def layer2(f1):
            if f1 not in h2_of:
                h = h1[w].copy()
                h[list(f1)] = alt1[r, list(f1)]
                r2, alt2 = tf32_flip_choices(h @ t2.T + b2, tf32_accumulation_bound(h[None], t2, b2)[0])
                h2_of[f1] = (r2, alt2, list(np.where(~np.isnan(alt2))[0]))
            return h2_of[f1]

        def candidates():                            # flip sets in order of their size, h1 choices first
            for nflips in range(1, len(amb1) + H + 1):
                produced = False
                for k1 in range(min(nflips, len(amb1)) + 1):
                    for f1 in itertools.combinations(amb1, k1):
                        r2, alt2, amb2 = layer2(f1)
                        for f2 in itertools.combinations(amb2, nflips - k1):
                            g = r2.copy()
                            g[list(f2)] = alt2[list(f2)]
                            produced = True
                            yield g
                if not produced:                     # no flip set of this size, hence none larger
                    return

        any_ambiguous = bool(amb1) or bool(layer2(())[2])
        tried, ok = 0, False
        if any_ambiguous:
            for g in itertools.islice(candidates(), TF32_MAX_COMBOS):
                tried += 1
                if (np.abs(segment_softmax(g @ t3.T + b3 + noise[w], segments) - got[w]) <= atol).all():
                    ok = True
                    break
        if not ok:
            unexplained.append((int(w), any_ambiguous, tried, float(np.abs(got[w] - want[w]).max())))
    assert not unexplained, ("%d of %d rows beyond %g are not TF32 rounding flips (row, has an ambiguous unit, "
                             "combinations tried, max |difference|): %s" % (len(unexplained), bad.size, atol,
                                                                            unexplained[:8]))
    return int(bad.size)
