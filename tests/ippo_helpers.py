"""Models and tables of IPPO's local critics (env.rollout_policy(..., critic=..., centralized_critic=False)): agent k's
critic reads obs_k alone, so the centralized critics' float64 models serve unchanged with [obs_k] as the observation
list (critic_helpers.CriticModel, rcritic_helpers.RecurrentModel); this module adds the seeded local critics, the
mirror of the MLP kernels' block table (LocalCriticShape, local_critic_smem_warps and local_critic_block_warps in
csrc/mpe_kernels.cu) and the recurrent kernel's programs."""
from critic_helpers import H, SMEM_OPTIN_BYTES, CriticModel, make_critic
from mappo_helpers import FEATURE_NORM, TANH
from mlp_programs import PROGRAMS, mlp_register_warps, mlp_smem_bytes, shapes_of
from rcritic_helpers import RCRITIC_PROGRAMS, RCRITIC_WARPS, make_rcritic

# LocalCriticRegisterException: (tag, MAPPO forms, warps) where MAPPO's register rule would spill
LOCAL_CRITIC_REGISTER_EXCEPTIONS = [
    ("simple", ("M",), 12),
    ("simple_push", ("M", "ME"), 12),
    ("simple_crypto", ("ME",), 12),
    ("simple_reference", ("ME",), 8),
    ("simple_spread_n4", ("M", "ME"), 8),
    ("simple_spread_n5", ("M",), 8),
    ("simple_adversary_n4", ("M", "ME"), 8),
]
# the recurrent local critic: the recurrent actor's programs, kRCriticWarps per block
RLOCAL_PROGRAMS, RLOCAL_WARPS = RCRITIC_PROGRAMS, RCRITIC_WARPS


def local_critic_bytes(obs_dim):
    """one local critic's weights: W1's fragments over obs_dim rounded up to 8 rows, W2, W3 (one n-tile), b1, b2, b3 [8]"""
    return 4 * (64 * ((obs_dim + 7) // 8) * 8 + 64 * 64 + 64 * 8 + 64 + 64 + 8)


def shared_ok(tag):
    """one shared local critic needs agents that observe alike"""
    return len(set(shapes_of(tag)[0])) == 1


def local_critic_smem_warps(tag, count):
    """warps whose tiles fit next to the actor and `count` local critics (1: one shared critic, agent 0's width)"""
    obs_dims, act_dims = shapes_of(tag)
    critics = local_critic_bytes(obs_dims[0]) if count == 1 else sum(local_critic_bytes(od) for od in obs_dims)
    fixed = mlp_smem_bytes(H, obs_dims, act_dims, 0) + critics
    per_warp = mlp_smem_bytes(H, obs_dims, act_dims, 1) - mlp_smem_bytes(H, obs_dims, act_dims, 0)
    return (SMEM_OPTIN_BYTES - fixed) // per_warp


def min_count(tag):
    """the smallest set a call may pass: one shared critic where the agents observe alike, else one per agent"""
    return 1 if shared_ok(tag) else len(shapes_of(tag)[0])


# the programs with the MLP local-critic kernels: every MAPPO program whose smallest set leaves room for a warp
LOCAL_PROGRAMS = tuple(t for t in PROGRAMS if local_critic_smem_warps(t, min_count(t)) >= 1)


def local_critic_block_cap(tag, episodes):
    """the compile-time cap: MAPPO's register rule or the exception, lowered to the smallest set's room"""
    form = "ME" if episodes else "M"
    r = None
    for t, forms, warps in LOCAL_CRITIC_REGISTER_EXCEPTIONS:
        if t == tag and form in forms:
            r = warps
    if r is None:
        r = mlp_register_warps(tag, H, episodes, True, True)
    return min(r, local_critic_smem_warps(tag, min_count(tag)))


def make_local_critics(obs_dims, mode, tanh, feature_norm, seed=5, eps=1e-5, device="cuda"):
    """"shared": one seeded critic on obs_dims[0] inputs; "per_agent": one per agent on its own obs_dim"""
    if mode == "shared":
        return make_critic([obs_dims[0]], tanh, feature_norm, seed=seed, eps=eps, device=device)
    return [make_critic([od], tanh, feature_norm, seed=seed + 6 + k, eps=eps, device=device)
            for k, od in enumerate(obs_dims)]


def local_models(critic, obs_dims):
    """agent k's float64 model of the kernel's recipe (CriticModel on [obs_dim_k]) and its unfolded module"""
    import torch
    from multiagent_particle_envs_b200.environment import mappo_actor_params
    mods = critic if isinstance(critic, list) else [critic] * len(obs_dims)
    models = []
    for k, m in enumerate(mods):
        params, tanh, fn, eps = mappo_actor_params([m], [obs_dims[k]], [1])
        net = ((FEATURE_NORM if fn else 0) | (TANH if tanh else 0), eps)
        models.append(CriticModel([t.to(torch.float32).cpu().numpy() for t in params[0]], net, [obs_dims[k]]))
    return models, mods


__all__ = ["LOCAL_CRITIC_REGISTER_EXCEPTIONS", "LOCAL_PROGRAMS", "RLOCAL_PROGRAMS", "RLOCAL_WARPS",
           "local_critic_block_cap", "local_critic_bytes", "local_critic_smem_warps", "local_models",
           "make_local_critics", "make_rcritic", "min_count", "shared_ok"]
