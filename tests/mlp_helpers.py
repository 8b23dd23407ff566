"""NumPy models of the two-hidden-layer in-kernel actor (env.rollout_policy with a Linear-ReLU-Linear-ReLU-Linear
policy): TF32 rounding as cvt.rna.tf32.f32 does it, Philox4x32-10, the Gumbel noise stream of act_dim logits, a float64
evaluation of the actor with or without the kernel's operand rounding, one softmax per action sub-space (movement,
utterance), and the accounting for its TF32 rounding flips."""
import itertools

import numpy as np

EXPLORE_TAG = 0x40000000


def tf32_rna(x):
    """fp32 -> TF32 (10 explicit mantissa bits) rounded to nearest, ties away from zero, returned as float32.  Adding
    half a TF32 unit to the magnitude bits and truncating rounds ties away from zero; a mantissa carry moves into the
    exponent as it should.  Inf and NaN pass unchanged."""
    b = np.asarray(x, dtype=np.float32).view(np.uint32)
    r = ((b.astype(np.uint64) + 0x1000) & 0xFFFFE000).astype(np.uint32)
    special = (b & 0x7F800000) == 0x7F800000
    return np.where(special, b, r).view(np.float32)


def tf32_rne(x):
    """fp32 -> TF32 rounded to nearest, ties to EVEN (what cvt.rna is not), as float32; finite inputs"""
    b = np.asarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    return (((b + 0xFFF + ((b >> 13) & 1)) & 0xFFFFE000).astype(np.uint32)).view(np.float32)


def tf32_tie(x, every=1):
    """x (float32) with every `every`-th entry (flat index) moved onto a TF32 rounding tie: the 13 bits below TF32 set
    to exactly half a unit, where ties-away and ties-to-even rounding part"""
    b = np.array(x, dtype=np.float32).view(np.uint32)
    pick = (np.arange(b.size) % every == 0).reshape(b.shape)
    return np.where(pick, (b & np.uint32(0xFFFFE000)) | np.uint32(0x1000), b).view(np.float32)


def dyadic_actor(rng, od=6, H=32, scale=2.0):
    """weights and observations on a 2^-4 grid: every sum is exact and every h1 / h2 value a short dyadic number, so no
    unit lies near a TF32 rounding boundary"""
    q = lambda *s: (np.round(rng.randn(*s) * scale * 16) / 16).astype(np.float32)        # noqa: E731
    params = (q(H, od) / 4, q(H) / 4, q(H, H) / 16, q(H) / 4, q(5, H) / 4, q(5) / 4)
    obs = q(32, od)
    return obs, params


def philox4x32_10(ctr, key):
    """Philox4x32-10 (Salmon et al., SC'11): ctr uint32 [..., 4], key (k0, k1) -> uint32 [..., 4]"""
    M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
    mask = np.uint64(0xFFFFFFFF)
    ctr = np.asarray(ctr, dtype=np.uint64)
    c = [ctr[..., j] for j in range(4)]
    k0, k1 = np.uint64(key[0]), np.uint64(key[1])
    for _ in range(10):
        p0 = np.uint64(M0) * c[0]
        p1 = np.uint64(M1) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & mask, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & mask]
        k0 = (k0 + np.uint64(W0)) & mask
        k1 = (k1 + np.uint64(W1)) & mask
    return np.stack(c, -1).astype(np.uint32)


def uniform_from_bits(bits):
    """u = ((bits >> 8) + 0.5) * 2^-24 with the sum rounded toward zero in fp32: exact below 2^23, above it the half
    does not fit in 24 bits and is dropped.  float32 in [2^-25, 1 - 2^-24]."""
    m = (np.asarray(bits, dtype=np.uint32) >> 8).astype(np.float64)
    s = np.where(m < 2 ** 23, m + 0.5, m)
    return (s * 2.0 ** -24).astype(np.float32)


def gumbel_noise(seed, epoch, world_index, t, agent, n_agents, n_logits=5, stride=2):
    """-log(-log u) of the `n_logits` logits of `agent` at step `t` for the given global world indices, float64.  Logit
    k uses word k mod 4 of Philox block b = k div 4, counter word 3 = EXPLORE_TAG | ((t * n_agents + agent) * stride + b);
    stride is 2 when every action vector of the scenario has at most 8 entries, else 4.  The defaults are the five
    movement logits."""
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


def actor_logits(obs, W1, b1, W2, b2, W3, b3, tf32=True):
    """float64 logits of the actor.  tf32=True rounds every tensor-core operand (observations, h1, h2, weights) to TF32
    as the kernel does; tf32=False evaluates the fp32 weights exactly."""
    f64 = np.float64
    rnd = tf32_rna if tf32 else (lambda a: np.asarray(a, dtype=np.float32))
    h1 = np.maximum(rnd(obs).astype(f64) @ rnd(W1).astype(f64).T + np.asarray(b1, f64), 0.0)
    h2 = np.maximum(rnd(h1).astype(f64) @ rnd(W2).astype(f64).T + np.asarray(b2, f64), 0.0)
    return rnd(h2).astype(f64) @ rnd(W3).astype(f64).T + np.asarray(b3, f64)


def softmax(z):
    e = np.exp(z - z.max(-1, keepdims=True))
    return e / e.sum(-1, keepdims=True)


def segment_softmax(z, segments=None):
    """one softmax per action sub-space: `segments` lists their widths in order (None: one softmax over the row)"""
    if segments is None:
        return softmax(z)
    assert sum(segments) == z.shape[-1], (segments, z.shape)
    bounds = np.cumsum([0] + list(segments))
    return np.concatenate([softmax(z[..., a:b]) for a, b in zip(bounds[:-1], bounds[1:])], -1)


# ---- accounting for TF32 rounding flips between the kernel and the float64 actor -------------------------------------
# actor_logits(tf32=True) rounds every tensor-core operand exactly as the kernel does, so the two can only differ through
# fp32 accumulation: in the logits by ~1e-7, and in a hidden layer where a unit's fp32 sum and the float64 sum fall on
# different sides of a TF32 rounding boundary -- h1 / h2 then round to neighbouring TF32 values, 2^-10 relative apart,
# and the row moves by up to a few 1e-4.  Every row beyond atol must be explained that way.
#
# Accumulation-error bound of one unit, sum_k a_k b_k + bias over K products (tf32_accumulation_bound): the operands
# have 11 significant bits, so every product is exact in fp32 and only the additions err.  The tensor cores add a whole
# k-tile of 8 products to the accumulator at once (aligned to the largest term, not sequential round-to-nearest), so
# the textbook K u S bound of a sequential fp32 sum (u = 2^-24, S = sum_k |a_k b_k| + |bias|, no partial sum exceeds S)
# does not apply as such.  tools/tf32_mma_error.cu measures the error of the kernel's exact mma.sync chain against the
# exact sum on actor-like operands: at most 2.0, 2.9, 3.3 and 4.1 u S for K = 8, 16, 32 and 64 (H100 SXM, 400 W, 2^19
# sums per K).  We allow 2 u S per k-tile plus 4 u S: (K/4 + 4) u S, i.e. 6, 8, 12 and 20 u S for those K -- 3 to 5
# times the measured worst case.
#
# Per row, a unit is ambiguous when relu(pre-activation) lies within the bound of a TF32 rounding boundary (units
# within the bound of zero are not: relu clips them to [0, bound], far below atol downstream).  Combinations of
# ambiguous units are enumerated layer by layer, in order of their number of flips: every choice of h1 flips, then h2
# recomputed -- and its ambiguity with it, so that an h1 flip too small to matter by itself can still carry an h2 unit
# across a boundary -- and every choice of h2 flips.
#
# How strict this is: at H = 64 most rows hold an ambiguous unit (a few per row, mostly small ones), so "has an
# ambiguous unit" alone rules out little there.  What does is the re-evaluation: a flip moves a row along one of a few
# fixed directions, so a change of the row in any other direction -- a wrong logit, a wrong lane, a row that no longer
# sums to one -- is not explained unless it happens to lie within atol of one of those directions.  A wrong logit that
# moves the row by 3e-5 can still pass in a sizeable fraction of rows at H = 64; by 3e-4 almost never.  A systematic
# defect moves many rows and is caught.
TF32_MAX_COMBOS = 2 ** 6


def tf32_accumulation_bound(a, b, bias):
    """per-unit bound on |fp32 tensor-core sum - exact sum| for rows a [m, K] (TF32 values) times weights b [N, K]"""
    K = a.shape[-1]
    return (K / 4.0 + 4.0) * 2.0 ** -24 * (np.abs(a) @ np.abs(b).T + np.abs(bias))


def tf32_flip_choices(pre, bound):
    """(relu(pre) rounded to TF32 as the model does, the other TF32 value a sum within `bound` of pre may round to --
    NaN where the unit is not ambiguous)"""
    f32 = np.float32
    r = tf32_rna(np.maximum(pre, 0.0).astype(f32)).astype(np.float64)
    lo = tf32_rna(np.maximum(pre - bound, 0.0).astype(f32)).astype(np.float64)
    hi = tf32_rna((pre + bound).astype(f32)).astype(np.float64)
    alt = np.where(lo != r, lo, np.where(hi != r, hi, np.nan))
    alt[pre <= bound] = np.nan
    return r, alt


def flipped(r, alt, flips):
    """the rounded row r with every unit of the groups in `flips` set to its alternative"""
    idx = [j for group in flips for j in group]
    g = r.copy()
    g[idx] = alt[idx]
    return g


def flip_candidates(first, next_layers):
    """The last layer's rounded row under every combination of TF32 rounding flips, in order of the number of flips,
    earlier layers' flips first (the enumeration the explainers share).  `first` is a layer of one row: (rounded row,
    alternatives, ambiguous groups), a group being a tuple of units that flip together.  Each of `next_layers` maps the
    previous layer's rounded row, flips applied, to the next layer of that row, so that its values and ambiguity follow
    the flips before it.  Stops at the first number of flips that no combination reaches, since none larger does."""
    cache = {}

    def layer(depth, prev):
        key = (depth, prev.tobytes())
        if key not in cache:
            cache[key] = next_layers[depth](prev)
        return cache[key]

    def rows(depth, lay, nflips):                    # every row of the last layer reached with exactly nflips flips
        r, alt, groups = lay
        if depth == len(next_layers):
            for f in itertools.combinations(groups, nflips):
                yield flipped(r, alt, f)
            return
        for k in range(min(nflips, len(groups)) + 1):
            for f in itertools.combinations(groups, k):
                yield from rows(depth + 1, layer(depth, flipped(r, alt, f)), nflips - k)

    for nflips in itertools.count(1):
        produced = False
        for g in rows(0, first, nflips):
            produced = True
            yield g
        if not produced:
            return


def relu_layer(r, alt):
    """a ReLU layer of one row for flip_candidates: every ambiguous unit flips by itself"""
    return r, alt, [(int(j),) for j in np.where(~np.isnan(alt))[0]]


def relu_next_layer(t, b):
    """flip_candidates' layer after a rounded ReLU row h: relu(h . t^T + b) and its ambiguity, one row at a time"""
    return lambda h: relu_layer(*tf32_flip_choices(h @ t.T + b, tf32_accumulation_bound(h[None], t, b)[0]))


def explain_tf32_mismatches(actions, obs, params, noise=0.0, atol=1e-5, segments=None):
    """Assert that every row of the kernel's `actions` [n, act_dim] that differs from segment_softmax(actor_logits(obs,
    *params, tf32=True) + noise, segments) by more than atol is a TF32 rounding flip (see above): it has an ambiguous h1
    or h2 unit, and rounding some combination of them the other way brings it within atol.  `segments`: the widths of
    the action sub-spaces, e.g. [5, 10], each with its own softmax; None: one softmax over the row.  At most
    TF32_MAX_COMBOS combinations per row; a row that needs more fails.  Returns the number of explained rows."""
    f64 = np.float64
    W1, b1, W2, b2, W3, b3 = [np.asarray(p, dtype=np.float32) for p in params]
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
        tried, ok = 0, False
        for g in itertools.islice(flip_candidates(relu_layer(h1[w], alt1[r]), [relu_next_layer(t2, b2)]),
                                  TF32_MAX_COMBOS):
            tried += 1
            if (np.abs(segment_softmax(g @ t3.T + b3 + noise[w], segments) - got[w]) <= atol).all():
                ok = True
                break
        if not ok:                                   # a row with an ambiguous unit has at least one candidate
            unexplained.append((int(w), tried > 0, tried, float(np.abs(got[w] - want[w]).max())))
    assert not unexplained, ("%d of %d rows beyond %g are not TF32 rounding flips (row, has an ambiguous unit, "
                             "combinations tried, max |difference|): %s" % (len(unexplained), bad.size, atol,
                                                                            unexplained[:8]))
    return int(bad.size)
