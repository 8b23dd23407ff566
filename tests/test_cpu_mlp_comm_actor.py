"""CPU checks of the two-hidden-layer actor's host side for scenarios with speaking or immovable agents: validation of
heads with act_dim_i outputs, the generalised Gumbel noise stream, the TF32 accounting with one softmax per action
sub-space, and the block-size cap the GPU tests mirror."""
import itertools

import numpy as np
import pytest

from helpers import make_product_env
import mlp_helpers
from mlp_helpers import (EXPLORE_TAG, explain_tf32_mismatches, gumbel_noise, philox4x32_10, segment_softmax, softmax,
                         tf32_rna, tf32_tie, uniform_from_bits)
from mlp_programs import mlp_register_rule

torch = pytest.importorskip("torch")


def _gumbel_noise_5(seed, epoch, world_index, t, agent, n_agents):
    """the five-logit stream as it was first defined: u_0..u_3 from block 0 and u_4 = word 0 of block 1, counter word 3
    = EXPLORE_TAG | ((t * A + i) * 2 + b)"""
    gw = np.asarray(world_index, dtype=np.uint64)
    key = (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    base = EXPLORE_TAG | ((t * n_agents + agent) * 2)
    words = []
    for b in (0, 1):
        ctr = np.stack([gw & np.uint64(0xFFFFFFFF), gw >> np.uint64(32), np.full_like(gw, epoch & 0xFFFFFFFF),
                        np.full_like(gw, base | b)], -1)
        words.append(philox4x32_10(ctr, key))
    bits = np.concatenate([words[0], words[1][:, :1]], 1)
    return -np.log(-np.log(uniform_from_bits(bits).astype(np.float64)))


@pytest.mark.parametrize("tag,obs_dims,act_dims", [("simple_speaker_listener", [3, 11], [3, 5]),
                                                   ("simple_reference", [21, 21], [15, 15])])
def test_heads_of_act_dim_outputs(tag, obs_dims, act_dims):
    from multiagent_particle_envs_b200.environment import mlp_actor_params
    nn = torch.nn
    shapes = make_product_env(tag, num_envs=64).world.native_shapes()          # device-less handle
    assert list(shapes.obs_dims) == obs_dims and list(shapes.act_dims) == act_dims
    H = 32
    mods = [nn.Sequential(nn.Linear(od, H), nn.ReLU(), nn.Linear(H, H), nn.ReLU(), nn.Linear(H, ad))
            for od, ad in zip(obs_dims, act_dims)]
    params, hidden = mlp_actor_params(mods, obs_dims, act_dims)
    assert hidden == H
    for p, od, ad in zip(params, obs_dims, act_dims):
        assert [tuple(t.shape) for t in p] == [(H, od), (H,), (H, H), (H,), (ad, H), (ad,)]
    tuples = [tuple(t.detach() for t in p) for p in params]
    assert mlp_actor_params(tuples, obs_dims, act_dims)[1] == H
    # a movement-only head on agent 0 (a speaker in both scenarios) is refused, naming the expected shapes
    five = [nn.Sequential(nn.Linear(obs_dims[0], H), nn.ReLU(), nn.Linear(H, H), nn.ReLU(), nn.Linear(H, 5))] + mods[1:]
    want = "W3 \\[%d, %d\\], b3 \\[%d\\]; got .*\\[5, %d\\], \\[5\\]" % (act_dims[0], H, act_dims[0], H)
    with pytest.raises(ValueError, match=want):
        mlp_actor_params(five, obs_dims, act_dims)
    with pytest.raises(ValueError, match=want):
        mlp_actor_params([tuples[0][:4] + (torch.zeros(5, H), torch.zeros(5))] + tuples[1:], obs_dims, act_dims)
    # without act_dims every head must have 5 outputs, as before
    if act_dims[0] != 5:
        with pytest.raises(ValueError, match="W3 \\[5, %d\\]" % H):
            mlp_actor_params(mods, obs_dims)


def test_generalised_gumbel_stream_keeps_the_five_logit_stream():
    seed, epoch, A = 0x1234_5678_9ABC, 3, 3
    gw = np.array([0, 1, 2, 31, 32, 2 ** 32 + 5, 2 ** 40 + 17], dtype=np.uint64)
    for t, i in itertools.product((0, 1, 7), range(A)):
        old = _gumbel_noise_5(seed, epoch, gw, t, i, A)
        assert np.array_equal(gumbel_noise(seed, epoch, gw, t, i, A), old)
        assert np.array_equal(gumbel_noise(seed, epoch, gw, t, i, A, n_logits=5, stride=2), old)
        # fewer logits: a prefix of block 0
        assert np.array_equal(gumbel_noise(seed, epoch, gw, t, i, A, n_logits=3), old[:, :3])
    # 15 logits at stride 4 (simple_reference): four blocks per agent and step, so agent 1's blocks start at 4, not 2
    s2 = gumbel_noise(seed, epoch, gw, 0, 1, 2, n_logits=15, stride=2)
    s4 = gumbel_noise(seed, epoch, gw, 0, 1, 2, n_logits=15, stride=4)
    assert s4.shape == (gw.size, 15)
    assert not np.array_equal(s2[:, :5], s4[:, :5])
    # agent 0 at step 0 starts at block 0 under either stride; its 15 logits use four distinct blocks
    a0 = gumbel_noise(seed, epoch, gw, 0, 0, 2, n_logits=15, stride=4)
    assert np.array_equal(a0, gumbel_noise(seed, epoch, gw, 0, 0, 2, n_logits=15, stride=2))
    assert len({a0[0, 4 * b:4 * b + 3].tobytes() for b in range(4)}) == 4


def _dyadic_actor(rng, od=6, H=32, ad=15, scale=2.0):
    """weights and observations on a 2^-4 grid: every sum is exact and no unit lies near a TF32 rounding boundary"""
    q = lambda *s: (np.round(rng.randn(*s) * scale * 16) / 16).astype(np.float32)        # noqa: E731
    return q(32, od), (q(H, od) / 4, q(H) / 4, q(H, H) / 16, q(H) / 4, q(ad, H) / 4, q(ad) / 4)


def _actions(obs, params, segs, h1_override=None):
    f64 = np.float64
    W1, b1, W2, b2, W3, b3 = params
    h1 = tf32_rna(np.maximum(tf32_rna(obs).astype(f64) @ tf32_rna(W1).astype(f64).T + b1, 0).astype(np.float32)).astype(f64)
    if h1_override is not None:
        h1[h1_override[0], h1_override[1]] = h1_override[2]
    h2 = tf32_rna(np.maximum(h1 @ tf32_rna(W2).astype(f64).T + b2, 0).astype(np.float32)).astype(f64)
    return segment_softmax(h2 @ tf32_rna(W3).astype(f64).T + b3, segs)


def test_segment_softmax():
    z = np.random.RandomState(0).randn(4, 15)
    p = segment_softmax(z, [5, 10])
    assert np.allclose(p[:, :5], softmax(z[:, :5])) and np.allclose(p[:, 5:], softmax(z[:, 5:]))
    assert np.array_equal(segment_softmax(z), softmax(z)) and np.array_equal(segment_softmax(z, [15]), softmax(z))
    with pytest.raises(AssertionError):
        segment_softmax(z, [5, 5])


def test_segmented_accounting_accepts_a_unit_on_a_tf32_midpoint_rounded_the_other_way():
    segs = [5, 10]
    obs, (W1, b1, W2, b2, W3, b3) = _dyadic_actor(np.random.RandomState(1))
    W1, b1, W2 = W1.copy(), b1.copy(), W2.copy()
    W1[0] = 0.0
    b1[0] = np.float32(1 + 2 ** -11)          # unit 0: pre-activation exactly on a TF32 tie
    W2[:, 0] = 1.0                            # make the flip visible in the actions
    params = (W1, b1, W2, b2, W3, b3)
    want = _actions(obs, params, segs)
    got = _actions(obs, params, segs, h1_override=(5, 0, 1.0))
    assert np.abs(got - want)[5].max() > 1e-4 and np.abs(got - want)[np.arange(32) != 5].max() == 0
    assert explain_tf32_mismatches(got, obs, params, segments=segs) == 1
    assert explain_tf32_mismatches(want, obs, params, segments=segs) == 0


def test_segmented_accounting_rejects_one_softmax_over_movement_and_utterance():
    """the comm logits normalised together with the movement logits, as a kernel that ignored the sub-spaces would"""
    segs = [5, 10]
    obs, params = _dyadic_actor(np.random.RandomState(2))
    right = _actions(obs, params, segs)
    assert explain_tf32_mismatches(right, obs, params, segments=segs) == 0
    joint = _actions(obs, params, None)
    assert np.abs(joint - right).max() > 1e-2
    with pytest.raises(AssertionError, match="not TF32 rounding flips"):
        explain_tf32_mismatches(joint, obs, params, segments=segs)
    # and the unsegmented accounting does not take the segmented actions either
    with pytest.raises(AssertionError, match="not TF32 rounding flips"):
        explain_tf32_mismatches(right, obs, params)


def test_block_cap_for_longer_action_vectors():
    """the general register rule with the largest action vector: 16 warps, or 12 at H = 64 for four or more agents, for
    5-entry vectors (simple, spread N=3, tag 3+1), 12 warps for simple_reference's 15-entry vectors at H = 64"""
    for H, A in itertools.product((32, 64), (1, 2, 3, 4)):
        assert mlp_register_rule(H, A) == mlp_register_rule(H, A, 5) == (12 if (H == 64 and A >= 4) else 16)
    assert [mlp_register_rule(64, 1), mlp_register_rule(64, 3), mlp_register_rule(64, 4), mlp_register_rule(32, 4)] == \
        [16, 16, 12, 16]
    # simple_speaker_listener (3, 5), simple_crypto (4), simple_adversary / simple_push (5), simple_reference (15)
    assert [mlp_register_rule(64, 2, 5), mlp_register_rule(64, 3, 4), mlp_register_rule(64, 3, 5),
            mlp_register_rule(64, 2, 15)] == [16, 16, 16, 12]
    assert mlp_register_rule(32, 2, 15) == 16


def _generic_actor(rng, od=18, H=64):
    r = lambda *s: rng.randn(*s).astype(np.float32)                                     # noqa: E731
    params = (tf32_tie(r(H, od) * 1.5 / od ** 0.5, 3), r(H) * 0.3, tf32_tie(r(H, H) * 1.5 / H ** 0.5, 3), r(H) * 0.3,
              r(5, H) * 1.5 / H ** 0.5, r(5) * 0.2)
    return rng.uniform(-1.5, 1.5, (256, od)).astype(np.float32), params


def test_accounting_without_segments_is_the_five_logit_accounting():
    """with one sub-space, given as [5] or as None, the accounting explains the same rows and rejects the same rows:
    rows moved by a rounding flip, by an unexplainable nudge and by a wrong, renormalised logit"""
    obs, params = _generic_actor(np.random.RandomState(5))
    z = mlp_helpers.actor_logits(obs, *params)
    got = softmax(z)
    # the actor with fp32 sums, as the tensor cores accumulate: some hidden units round the other way
    f32 = np.float32
    W1, b1, W2, b2, W3, b3 = params
    h1 = tf32_rna(np.maximum(tf32_rna(obs) @ tf32_rna(W1).T + b1, 0).astype(f32))
    h2 = tf32_rna(np.maximum(h1 @ tf32_rna(W2).T + b2, 0).astype(f32))
    fp32 = softmax((h2 @ tf32_rna(W3).T + b3).astype(np.float64))
    n_ref = explain_tf32_mismatches(fp32, obs, params)
    assert n_ref > 0
    for acts, n in ((got, 0), (fp32, n_ref)):
        assert explain_tf32_mismatches(acts, obs, params) == n
        assert explain_tf32_mismatches(acts, obs, params, segments=[5]) == n
    nudged = got.copy()
    nudged[31, 4] += 1e-4
    wrong = got.copy()
    zz = z[40].copy()
    zz[zz.argmax()] += 4e-3
    wrong[40] = softmax(zz)
    for acts in (nudged, wrong):
        with pytest.raises(AssertionError, match="not TF32 rounding flips"):
            explain_tf32_mismatches(acts, obs, params)
        with pytest.raises(AssertionError, match="not TF32 rounding flips"):
            explain_tf32_mismatches(acts, obs, params, segments=[5])
