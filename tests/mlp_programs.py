"""The 17 programs the two-hidden-layer in-kernel actor is built for, the mirror of its block-size cap, and the fixtures
the GPU tests of that actor share (seeded actors, twin envs)."""
import functools

from helpers import CONFIGS, VARIANTS, make_product_env

# The entity-count variants, tag -> (scenario name, scenario kwargs)
VARIANT_PROGRAMS = {tag: CONFIGS[tag] if tag in CONFIGS else VARIANTS[tag]
                    for tag in ("simple_spread_n2", "simple_spread_n4", "simple_spread_n5", "simple_spread_n6",
                                "simple_tag_1v1", "simple_tag_2v1", "simple_tag_4v2", "simple_tag_6v2", "simple_adversary_n4")}
# every program mpe_policy_mlp_rollout_kernel is built for (MlpBuilt): all but simple_world_comm
PROGRAMS = {**{t: s for t, s in CONFIGS.items() if t != "simple_world_comm"}, **VARIANT_PROGRAMS}
assert len(PROGRAMS) == 17

# Against the float64 actor with the kernel's TF32 operand rounding every row beyond TIGHT_ATOL must be a TF32 rounding
# flip (mlp_helpers.explain_tf32_mismatches); against the unrounded float64 actor the probabilities stay within
# LOOSE_MAX (see tests/test_gpu_mlp_policy.py)
TIGHT_ATOL = 1e-5
LOOSE_MAX = 5e-3


@functools.lru_cache(maxsize=None)
def shapes_of(tag):
    """(obs_dims, act_dims) of a program, from its shape-only handle"""
    s = make_product_env(tag, num_envs=1).world.native_shapes()
    return tuple(s.obs_dims), tuple(s.act_dims)


# ---- block-size cap: mlp_block_warps in csrc/mpe_kernels.cu ------------------------------------------------------------
# The dynamic shared memory one block may opt in to on H100 (cudaDevAttrMaxSharedMemoryPerBlockOptin)
SMEM_OPTIN_BYTES = 232448

# The forms, in the kernel's order (episodes | kind << 1, kind 0 softmax, 1 categorical, 2 MAPPO's actor): softmax,
# softmax episodes, categorical, categorical episodes, MAPPO, MAPPO episodes.  MAPPO's forms exist at H = 64 only.
FORMS = ("S", "E", "C", "CE", "M", "ME")
# MlpRegisterException: (tag, H, forms, warps) where the general rule would spill (12 warps leave 168 registers per
# thread, 8 leave 255)
REGISTER_EXCEPTIONS = [
    ("simple_spread_n2", 64, FORMS, 12),
    ("simple_tag_1v1", 64, FORMS, 12),
    ("simple_tag_2v1", 64, FORMS, 12),
    ("simple_spread_n6", 64, FORMS, 8),
    ("simple_spread_n6", 32, FORMS, 12),
    ("simple_tag_4v2", 32, FORMS, 12),
    ("simple_tag_6v2", 32, FORMS, 8),
    ("simple_speaker_listener", 64, ("E", "CE", "M", "ME"), 12),
    ("simple_adversary", 64, ("E", "CE", "M", "ME"), 12),
    ("simple_reference", 64, ("E", "CE"), 8),
    ("simple_tag_4v2", 64, ("E", "CE"), 8),
    ("simple_spread_n3", 64, ("E", "C", "CE", "M", "ME"), 12),
    ("simple_push", 64, ("C", "CE"), 12),
    ("simple_crypto", 64, ("CE", "M"), 12),
    ("simple_spread_n4", 64, ("CE",), 8),
]
# one exception per (program, H), as in the kernel, so that no kernel matches two
assert len({(tag, H) for tag, H, _, _ in REGISTER_EXCEPTIONS}) == len(REGISTER_EXCEPTIONS)


def mlp_register_rule(H, n_agents, max_act_dim=5):
    """the general register rule: 16 warps, or 12 at H = 64 for four or more agents or an action vector longer than 8
    entries (simple_reference: 15)"""
    return 12 if (H == 64 and (n_agents >= 4 or max_act_dim > 8)) else 16


def mlp_register_warps(tag, H, episodes=False, categorical=False, mappo=False):
    """mlp_register_warps: the general rule, or the exception for this program, H and form"""
    assert not mappo or (categorical and H == 64), "MAPPO's actor: categorical, H = 64"
    form = FORMS[int(episodes) | (2 if mappo else int(categorical)) << 1]
    for t, h, forms, warps in REGISTER_EXCEPTIONS:
        if (t, h) == (tag, H) and form in forms:
            return warps
    obs_dims, act_dims = shapes_of(tag)
    return mlp_register_rule(H, len(obs_dims), max(act_dims))


def mlp_smem_bytes(H, obs_dims, act_dims, warps):
    """MlpShape in csrc/mpe_kernels.cu: every agent's TF32 B fragments of W1 (obs_dim rounded up to 8 rows), W2 and W3
    (act_dim rounded up to 8 columns) plus b1, b2, b3, then per warp an observation tile (odd row pitch in store units)
    and a 32 x (max NOUT + 1) logit tile"""
    nt = H // 8
    nout = [(ad + 7) // 8 * 8 for ad in act_dims]
    weights = sum(64 * ((od + 7) // 8) * nt + 64 * nt * nt + 8 * nt * no + 2 * H + no for od, no in zip(obs_dims, nout))

    def pitch(od):
        unit = 2 if od % 2 == 0 else 1
        return ((od // unit) | 1) * unit

    obs_tile = (max(32 * pitch(od) for od in obs_dims) + 3) & ~3
    warp = (obs_tile + 32 * (max(nout) + 1) + 3) & ~3
    return 4 * (weights + warps * warp)


def mlp_block_cap(tag, H, episodes=False, categorical=False, mappo=False):
    """mlp_block_warps: the register cap lowered to the most warps whose tiles fit in shared memory next to the
    weights"""
    obs_dims, act_dims = shapes_of(tag)
    cap = mlp_register_warps(tag, H, episodes, categorical, mappo)
    while mlp_smem_bytes(H, obs_dims, act_dims, cap) > SMEM_OPTIN_BYTES:
        cap -= 1
    return cap


# ---- GPU fixtures -------------------------------------------------------------------------------------------------------
def make_policies(obs_dims, act_dims, H, seed=3):
    """seeded actors; every third weight on a TF32 rounding tie, so a rounding mode other than ties-away fails"""
    import torch
    from mlp_helpers import tf32_tie
    g = torch.Generator(device="cuda").manual_seed(seed)
    ties = lambda W: torch.as_tensor(tf32_tie(W.cpu().numpy(), 3), device="cuda")   # noqa: E731
    pols = []
    for od, ad in zip(obs_dims, act_dims):
        r = lambda *s: torch.randn(*s, device="cuda", generator=g)   # noqa: E731
        pols.append((ties(r(H, od) * 1.5 / od ** 0.5), r(H) * 0.3, ties(r(H, H) * 1.5 / H ** 0.5), r(H) * 0.3,
                     ties(r(ad, H) * 1.5 / H ** 0.5), r(ad) * 0.2))
    return pols


def as_sequential(pols):
    import torch
    mods = []
    for W1, b1, W2, b2, W3, b3 in pols:
        H = W1.shape[0]
        m = torch.nn.Sequential(torch.nn.Linear(W1.shape[1], H), torch.nn.ReLU(), torch.nn.Linear(H, H), torch.nn.ReLU(),
                                torch.nn.Linear(H, W3.shape[0])).cuda()
        with torch.no_grad():
            for lin, W, b in ((m[0], W1, b1), (m[2], W2, b2), (m[4], W3, b3)):
                lin.weight.copy_(W)
                lin.bias.copy_(b)
        mods.append(m)
    return mods


def twins(tag, n, seed=9, **kw):
    a = make_product_env(tag, num_envs=n, seed=seed, **kw)
    b = make_product_env(tag, num_envs=n, seed=seed, **kw)
    a.reset()
    b.reset()
    return a, b


def state(env):
    nw = env.world.native
    return [nw.agent_pv.clone(), nw.lm_p.clone(), nw.comm.clone(), nw.goal.clone()]
