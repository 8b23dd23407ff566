"""NumPy model of MAPPO's centralized critic in the in-kernel rollout (env.rollout_policy(..., critic=...),
mpe_rollout_policy_mappo_critic): the float64 evaluation of the folded critic with the kernel's recipe (MappoModel's, on
share_obs), the accounting for every value outside the flip-free bound by TF32 rounding flips of the normalised
operands, seeded critics, and the mirror of the critic kernels' block table (CriticShape and critic_block_warps in
csrc/mpe_kernels.cu)."""
import itertools

import numpy as np

from mappo_helpers import MAPPO_MAX_COMBOS, U, MappoModel, ambiguous_groups, flip_choices, next_layer, norm_error_bound
from mlp_helpers import flip_candidates, tf32_accumulation_bound, tf32_rna
from mlp_programs import PROGRAMS, mlp_register_warps, mlp_smem_bytes, shapes_of

H = 64
# against the unfolded float64 critic every value stays within LOOSE (TF32 operands through three layers)
LOOSE = 2e-2


def share_obs(obs_list):
    """MAPPO's share_obs with use_centralized_V: every agent's observation [..., obs_dim_i] concatenated in agent order"""
    return np.concatenate([np.asarray(o, np.float64) for o in obs_list], axis=-1)


class CriticModel(MappoModel):
    """the kernel's recipe in float64 for one critic (params: its folded float32 (W1, b1, W2, b2, W3, b3)).  Layer 1
    sums the agents' k-slices, each zero-padded to whole k-tiles of 8: its accumulation bound counts the padded width."""

    def __init__(self, params, net, obs_dims):
        super().__init__(params, net)
        self.k1 = sum((od + 7) // 8 * 8 for od in obs_dims)

    def hidden(self, x_rounded, layer):
        if layer != 0:
            return super().hidden(x_rounded, layer)
        from mappo_helpers import activation, layer_norm
        t, b = self.t[0], self.b[0]
        p = x_rounded @ t.T + b
        a = activation(p, self.tanh)
        ea = (self.k1 / 4.0 + 4.0) * U * (np.abs(x_rounded) @ np.abs(t).T + np.abs(b)) + \
            (2 * U * np.abs(a) if self.tanh else 0.0)
        return layer_norm(a, self.eps), norm_error_bound(a, ea, self.eps)

    def values(self, x):
        """(V [m], the flip-free bound on |kernel - V| [m]) of share_obs rows x [m, D]"""
        rnd = lambda v: tf32_rna(v.astype(np.float32)).astype(np.float64)   # noqa: E731
        x0 = rnd(self.input(x)[0])
        x1 = rnd(self.hidden(x0, 0)[0])
        x2 = rnd(self.hidden(x1, 1)[0])
        return self.logits(x2)[:, 0], tight_bound(self, x2)


def tight_bound(model, x2):
    """the fp32 accumulation error of layer 3 on the TF32 operands x2 [m, 64], plus a few ulps of the value"""
    v = x2 @ model.t[2].T + model.b[2]
    return tf32_accumulation_bound(x2, model.t[2], model.b[2])[:, 0] + 4 * U * np.abs(v[:, 0])


def explain_value_mismatches(got, x, model):
    """Assert that every value got [m] farther than the flip-free bound from the model on share_obs x [m, D] is the
    model's value, within that bound, under a combination of TF32 rounding flips of x0 (with the input LayerNorm), x1
    and x2 (mappo_helpers' ambiguity and enumeration).  Returns the number of rows explained by a flip."""
    v, tb = model.values(x)
    bad = np.where(np.abs(got - v) > tb)[0]
    x0v, e0 = model.input(x)
    flips, unexplained = 0, []
    for w in bad:
        if e0 is not None:
            r0, alt0 = flip_choices(x0v[w], e0[w])
        else:
            r0, alt0 = tf32_rna(x0v[w].astype(np.float32)).astype(np.float64), np.full(x0v.shape[1], np.nan)
        first = (r0, alt0, ambiguous_groups(x0v[w], alt0))
        ok, tried = False, 0
        for g in itertools.islice(flip_candidates(first, [next_layer(model, 0), next_layer(model, 1)]), MAPPO_MAX_COMBOS):
            tried += 1
            if abs(float(model.logits(g[None])[0, 0]) - float(got[w])) <= tight_bound(model, g[None])[0]:
                ok = True
                break
        if ok:
            flips += 1
        else:
            unexplained.append((int(w), float(got[w]), float(v[w]), float(tb[w]), tried))
    assert not unexplained, ("%d of %d values are not TF32 rounding flips of the normalised operands (row, kernel, "
                             "model, bound, combinations tried): %s" % (len(unexplained), bad.size, unexplained[:8]))
    return flips


def module_values(module, x):
    """the user's unfolded critic in float64 on the CPU, [m]"""
    from mappo_helpers import module_logits
    return module_logits(module, x)[:, 0]


def make_critic(obs_dims, tanh, feature_norm, seed=5, eps=1e-5, device="cuda"):
    """one seeded MAPPO critic over share_obs (non-trivial LayerNorm affines, every third weight on a TF32 tie)"""
    from mappo_helpers import make_mappo_actors
    return make_mappo_actors([int(sum(obs_dims))], [1], tanh, feature_norm, seed=seed, eps=eps, device=device)[0]


# ---- the block table: CriticShape, critic_smem_warps, critic_block_warps -------------------------------------------------
SMEM_OPTIN_BYTES = 232448
# CriticRegisterException: (tag, MAPPO forms, warps)
CRITIC_REGISTER_EXCEPTIONS = [
    ("simple", ("M",), 12),
    ("simple_push", ("M", "ME"), 12),
    ("simple_crypto", ("ME",), 12),
    ("simple_spread_n4", ("M", "ME"), 8),
    ("simple_adversary_n4", ("M", "ME"), 8),
]


def critic_bytes(obs_dims):
    """one critic's weights: W1's fragments per agent (obs_dim_i rounded up to 8 rows), W2, W3 (one n-tile), b1, b2,
    b3 [8]"""
    return 4 * (sum(64 * ((od + 7) // 8) * 8 for od in obs_dims) + 64 * 64 + 64 * 8 + 64 + 64 + 8)


def critic_smem_warps(tag, count):
    obs_dims, act_dims = shapes_of(tag)
    fixed = mlp_smem_bytes(H, obs_dims, act_dims, 0) + count * critic_bytes(obs_dims)
    per_warp = mlp_smem_bytes(H, obs_dims, act_dims, 1) - mlp_smem_bytes(H, obs_dims, act_dims, 0)
    return (SMEM_OPTIN_BYTES - fixed) // per_warp


# every MAPPO program with room for one shared critic and a warp: all but simple_spread N=6 and simple_tag 6+2
CRITIC_PROGRAMS = tuple(t for t in PROGRAMS if t not in ("simple_spread_n6", "simple_tag_6v2"))


def critic_block_cap(tag, episodes):
    """the compile-time cap: MAPPO's register rule or the critic's exception, lowered to one shared critic's room"""
    form = "ME" if episodes else "M"
    r = None
    for t, forms, warps in CRITIC_REGISTER_EXCEPTIONS:
        if t == tag and form in forms:
            r = warps
    if r is None:
        r = mlp_register_warps(tag, H, episodes, True, True)
    return min(r, critic_smem_warps(tag, 1))
