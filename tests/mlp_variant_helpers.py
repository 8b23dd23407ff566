"""The entity-count variants of simple_spread, simple_tag and simple_adversary that the two-hidden-layer in-kernel actor
is built for, and the mirror of its block-size cap with the shared-memory limit those programs reach."""
from helpers import CONFIGS, NO_BENCHMARK, VARIANTS
from mlp_comm_helpers import mlp_block_cap

# tag -> (scenario name, scenario kwargs)
PROGRAMS = {
    "simple_spread_n2": ("simple_spread", {"num_agents": 2}),
    "simple_spread_n4": ("simple_spread", {"num_agents": 4}),
    "simple_spread_n5": ("simple_spread", {"num_agents": 5}),
    "simple_spread_n6": CONFIGS["simple_spread_n6"],
    **{tag: VARIANTS[tag] for tag in ("simple_tag_1v1", "simple_tag_2v1", "simple_tag_4v2", "simple_tag_6v2",
                                      "simple_adversary_n4")},
}

# The dynamic shared memory one block may opt in to on H100 (cudaDevAttrMaxSharedMemoryPerBlockOptin)
SMEM_OPTIN_BYTES = 232448

# (tag, H) -> warps per block where mlp_comm_helpers.mlp_block_cap's would spill: the MlpRegisterWarps specialisations
# in csrc/mpe_kernels.cu (12 warps leave 168 registers per thread, 8 leave 255)
REGISTER_WARPS = {
    ("simple_spread_n2", 64): 12, ("simple_tag_1v1", 64): 12, ("simple_tag_2v1", 64): 12, ("simple_spread_n6", 64): 8,
    ("simple_spread_n6", 32): 12, ("simple_tag_4v2", 32): 12, ("simple_tag_6v2", 32): 8,
}


def make_variant_env(tag, **kw):
    from multiagent_particle_envs_b200 import make_env
    name, skw = PROGRAMS[tag]
    kw.update(skw)
    return make_env(name, benchmark=(name not in NO_BENCHMARK), **kw)


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


def mlp_register_cap(tag, H, obs_dims, act_dims):
    """mlp_register_warps: mlp_comm_helpers.mlp_block_cap, or REGISTER_WARPS where that spills"""
    return REGISTER_WARPS.get((tag, H), mlp_block_cap(H, len(obs_dims), max(act_dims)))


def mlp_variant_cap(tag, H, obs_dims, act_dims):
    """mlp_block_warps: the register cap lowered to the most warps whose tiles fit in shared memory next to the
    weights"""
    cap = mlp_register_cap(tag, H, obs_dims, act_dims)
    while mlp_smem_bytes(H, obs_dims, act_dims, cap) > SMEM_OPTIN_BYTES:
        cap -= 1
    return cap
