"""CPU checks of the block-size cap mirror of the two-hidden-layer actor (mlp_programs.mlp_block_cap): today's
caps for the programs built before the entity-count variants, and a shared-memory footprint within the per-block
opt-in limit for the variants, computed from the shape-only handle's observation and action widths."""
import pytest

from helpers import make_product_env
from mlp_programs import (SMEM_OPTIN_BYTES, mlp_block_cap, mlp_register_rule, mlp_register_warps,
                          mlp_smem_bytes)
from mlp_programs import VARIANT_PROGRAMS as PROGRAMS

pytest.importorskip("torch")

EXISTING = ("simple", "simple_spread_n3", "simple_tag", "simple_speaker_listener", "simple_reference", "simple_crypto",
            "simple_adversary", "simple_push")


@pytest.mark.parametrize("tag", EXISTING)
@pytest.mark.parametrize("H", [32, 64])
def test_existing_programs_keep_their_cap(tag, H):
    shapes = make_product_env(tag, num_envs=64).world.native_shapes()          # device-less handle
    obs_dims, act_dims = list(shapes.obs_dims), list(shapes.act_dims)
    want = mlp_register_rule(H, len(obs_dims), max(act_dims))
    assert mlp_block_cap(tag, H) == want
    assert mlp_smem_bytes(H, obs_dims, act_dims, want) <= SMEM_OPTIN_BYTES


@pytest.mark.parametrize("tag", list(PROGRAMS))
@pytest.mark.parametrize("H", [32, 64])
def test_variant_cap_fits_shared_memory(tag, H):
    shapes = make_product_env(tag, num_envs=64).world.native_shapes()          # device-less handle
    obs_dims, act_dims = list(shapes.obs_dims), list(shapes.act_dims)
    assert act_dims == [5] * len(obs_dims)
    cap = mlp_block_cap(tag, H)
    register_cap = mlp_register_warps(tag, H)
    assert 1 <= cap <= register_cap
    assert mlp_smem_bytes(H, obs_dims, act_dims, cap) <= SMEM_OPTIN_BYTES
    if cap < register_cap:                                   # shared memory binds: one more warp does not fit
        assert mlp_smem_bytes(H, obs_dims, act_dims, cap + 1) > SMEM_OPTIN_BYTES


def test_shared_memory_binds_only_for_the_largest_programs():
    """the footprints the kernel's static_asserts pin at H = 64: spread N=6's 171 KB of weights leave room for 9 warps
    (its registers allow 8), tag 6+2's 212 KB for 3; shared memory binds for no other (program, H)"""
    binding = {}
    for tag in PROGRAMS:
        shapes = make_product_env(tag, num_envs=64).world.native_shapes()
        od, ad = list(shapes.obs_dims), list(shapes.act_dims)
        for H in (32, 64):
            if mlp_smem_bytes(H, od, ad, mlp_register_warps(tag, H)) > SMEM_OPTIN_BYTES:
                binding[tag, H] = (mlp_smem_bytes(H, od, ad, 0), mlp_block_cap(tag, H))
        if tag == "simple_spread_n6":
            assert mlp_smem_bytes(64, od, ad, 0) == 175296
            assert mlp_smem_bytes(64, od, ad, 9) <= SMEM_OPTIN_BYTES < mlp_smem_bytes(64, od, ad, 10)
            assert mlp_block_cap(tag, 64) == 8
    assert binding == {("simple_tag_6v2", 64): (217344, 3)}
