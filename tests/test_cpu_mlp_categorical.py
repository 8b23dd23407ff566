"""CPU checks of the categorical form of the two-hidden-layer actor (env.rollout_policy(..., action_mode="categorical")):
the new C entry points are declared and bound, the NumPy models the GPU tests judge the kernel by (log-probability,
Gumbel arg-max, one-hot replay) agree with independent formulations, the flip accounting explains what a TF32 rounding
flip or the Gumbel gap explains and nothing else, and the refusals that need no device."""
import os
import re

import numpy as np
import pytest

from helpers import make_product_env
from mlp_categorical_helpers import (GUMBEL_GAP, bounds, categorical_pick, explain_categorical_mismatches, log_softmax_at,
                                     one_hot, split_pick_noise)
from mlp_helpers import (EXPLORE_TAG, actor_logits, dyadic_actor, gumbel_noise, philox4x32_10, segment_softmax, tf32_rna,
                         uniform_from_bits)

torch = pytest.importorskip("torch")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRY_POINTS = ("mpe_rollout_policy_mlp_categorical", "mpe_rollout_policy_mlp_categorical_episodes")


def test_categorical_entry_points_are_declared_and_bound():
    import ctypes
    from multiagent_particle_envs_b200 import _lib
    header = open(os.path.join(ROOT, "include", "mpe_b200.h")).read()
    declared = set(re.findall(r"MPE_API[^;(]*?\b(mpe_[a-z_]+)\s*\(", header))
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in ENTRY_POINTS:
        assert name in declared and name in _lib.EXPORTED_SYMBOLS and hasattr(lib, name), name
    # the parameters of the default form, with the int32 index records in place of the float action records and the
    # log-probabilities next to the per-step rewards
    for name, base in zip(ENTRY_POINTS, ("mpe_rollout_policy_mlp", "mpe_rollout_policy_mlp_episodes")):
        got, want = _lib._SIGNATURES[name][1], list(_lib._SIGNATURES[base][1])
        rew_steps = 19 if base == "mpe_rollout_policy_mlp" else 22
        assert got == want[:rew_steps + 1] + [_lib._P] + want[rew_steps + 1:], name
    assert _lib.MPE_ABI_VERSION == 1


@pytest.mark.parametrize("segs", [[5], [3], [5, 10], [5, 4]])
def test_log_probability_model_is_scipy_log_softmax(segs):
    from scipy.special import log_softmax
    rng = np.random.RandomState(1)
    z = rng.randn(4096, sum(segs)) * 3.0
    k = np.stack([rng.randint(0, b - a, 4096) for a, b in bounds(segs)], -1)
    want = sum(np.take_along_axis(log_softmax(z[:, a:b], -1), k[:, s:s + 1], 1)[:, 0]
               for s, (a, b) in enumerate(bounds(segs)))
    np.testing.assert_allclose(log_softmax_at(z, k, segs), want, rtol=0, atol=1e-12)


def _five_logit_noise(seed, epoch, world_index, t, agent, n_agents):
    """the five movement logits' Gumbel noise: u_0..u_3 = words 0-3 of block 0, u_4 = word 0 of block 1, counter
    (world index low, high, epoch, EXPLORE_TAG | ((t * A + i) * 2 + b)), key (seed low, high)"""
    gw = np.asarray(world_index, dtype=np.uint64)
    key = (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    word3 = EXPLORE_TAG | ((t * n_agents + agent) * 2)
    ctr = np.stack([gw & np.uint64(0xFFFFFFFF), gw >> np.uint64(32), np.full_like(gw, epoch & 0xFFFFFFFF),
                    np.full_like(gw, word3)], -1)
    block0 = philox4x32_10(ctr, key)
    ctr[:, 3] = word3 | 1
    block1 = philox4x32_10(ctr, key)
    u = uniform_from_bits(np.concatenate([block0, block1[:, :1]], 1)).astype(np.float64)
    return -np.log(-np.log(u))


@pytest.mark.parametrize("segs,stride", [([5], 2), ([3], 2), ([5, 10], 4), ([5, 3], 2)])
def test_gumbel_argmax_model_is_the_argmax_of_the_gumbel_softmax_sample(segs, stride):
    """categorical_pick(z + g) per sub-space is the arg-max of segment_softmax(z + g), the default mode's sample, with g
    the exploration stream of mlp_helpers.gumbel_noise (for five logits: words 0-3 of Philox block 0 and word 0 of block
    1, written out below)"""
    n, A = 4096, 3
    rng = np.random.RandomState(2)
    z = rng.randn(n, sum(segs))
    for t, i in ((0, 0), (7, 2)):
        g = gumbel_noise(99, 3, np.arange(n) + 10 ** 6, t, i, A, n_logits=sum(segs), stride=stride)
        if segs == [5]:
            np.testing.assert_array_equal(g, _five_logit_noise(99, 3, np.arange(n) + 10 ** 6, t, i, A))
        k = categorical_pick(z + g, segs)
        sample = segment_softmax(z + g, segs)
        for s, (a, b) in enumerate(bounds(segs)):
            np.testing.assert_array_equal(k[:, s], np.argmax(sample[:, a:b], -1))
        # the picks are distributed as softmax(z): over many draws of one row the frequencies approach it
    zz = np.tile(np.array([[0.5, -1.0, 1.2]]), (200000, 1))
    g = gumbel_noise(5, 0, np.arange(200000), 0, 0, 1, n_logits=3, stride=2)
    freq = np.bincount(categorical_pick(zz + g, [3])[:, 0], minlength=3) / 200000.0
    np.testing.assert_allclose(freq, segment_softmax(zz[:1])[0], atol=5e-3)


def test_ties_go_to_the_lowest_index_and_one_hot_inverts_the_pick():
    z = np.array([[1.0, 3.0, 3.0, 0.0, 0.0, 2.0, 2.0, 2.0]])
    k = categorical_pick(z, [5, 3])
    assert k.tolist() == [[1, 0]]
    assert one_hot(k, [5, 3]).tolist() == [[0, 1, 0, 0, 0, 1, 0, 0]]
    rng = np.random.RandomState(3)
    k = np.stack([rng.randint(0, 5, 100), rng.randint(0, 10, 100)], -1)
    np.testing.assert_array_equal(categorical_pick(one_hot(k, [5, 10]), [5, 10]), k)


# ---- explain_categorical_mismatches on synthetic actors (no GPU) -----------------------------------------------------
def _logits(obs, params, h1_override):
    """actor_logits with one rounded h1 entry, (row, unit, value), replaced"""
    f64 = np.float64
    W1, b1, W2, b2, W3, b3 = params
    h1 = tf32_rna(np.maximum(tf32_rna(obs).astype(f64) @ tf32_rna(W1).astype(f64).T + b1, 0).astype(np.float32)).astype(f64)
    h1[h1_override[0], h1_override[1]] = h1_override[2]
    h2 = tf32_rna(np.maximum(h1 @ tf32_rna(W2).astype(f64).T + b2, 0).astype(np.float32)).astype(f64)
    return h2 @ tf32_rna(W3).astype(f64).T + b3


def test_accounting_explains_a_pick_moved_by_a_tf32_flip_and_one_within_the_gumbel_gap():
    obs, (W1, b1, W2, b2, W3, b3) = dyadic_actor(np.random.RandomState(1))
    # unit 0: pre-activation 1 + 2^-11 exactly (a TF32 tie); the model rounds it up to 1 + 2^-10, the "kernel" rounds
    # row 5's down to 1
    W1, b1, W2 = W1.copy(), b1.copy(), W2.copy()
    W1[0] = 0.0
    b1[0] = np.float32(1 + 2 ** -11)
    W2[:, 0] = 1.0                          # make the flip visible in the logits
    params, segs = (W1, b1, W2, b2, W3, b3), [5]
    z = actor_logits(obs, *params)
    zk = _logits(obs, params, (5, 0, 1.0))
    noise = np.zeros_like(z)
    noise[5], pick5, half = split_pick_noise(z[5], zk[5])
    assert half > 1e-4                      # the pick moves, and by more than the Gumbel gap
    a, b = np.argsort(z[3])[::-1][:2]       # row 3: the runner-up within the Gumbel gap of the pick
    noise[3, b] = z[3, a] - z[3, b] - GUMBEL_GAP / 2
    k = categorical_pick(z + noise, segs)
    logp = log_softmax_at(z, k, segs)
    assert explain_categorical_mismatches(k, logp, obs, params, segs, noise=noise) == (0, 0)
    assert k[5, 0] != pick5 and k[3, 0] == a
    k[5, 0], k[3, 0] = pick5, b
    logp = log_softmax_at(z, k, segs)
    logp[5] = log_softmax_at(zk[5:6], k[5:6], segs)[0]
    assert explain_categorical_mismatches(k, logp, obs, params, segs, noise=noise) == (1, 1)


def test_accounting_rejects_a_wrong_pick_and_a_wrong_log_probability():
    obs, params = dyadic_actor(np.random.RandomState(2))
    segs = [5]
    z = actor_logits(obs, *params)
    k = categorical_pick(z, segs)
    logp = log_softmax_at(z, k, segs)
    assert explain_categorical_mismatches(k, logp, obs, params, segs) == (0, 0)
    bad = k.copy()
    bad[7, 0] = np.argmin(z[7])             # with the model's log-probability of that pick
    with pytest.raises(AssertionError, match="neither TF32 rounding flips nor within the Gumbel gap"):
        explain_categorical_mismatches(bad, log_softmax_at(z, bad, segs), obs, params, segs)
    wrong = logp.copy()
    wrong[7] += 1e-3
    with pytest.raises(AssertionError, match=r"\(7, "):
        explain_categorical_mismatches(k, wrong, obs, params, segs)


def test_refusals_without_a_device():
    """action_mode and record_log_probs are checked before anything else; the one-hidden-layer actor has no
    categorical form"""
    nn = torch.nn
    env = make_product_env("simple_spread_n3", num_envs=64)
    obs_dims = env.world.native_shapes().obs_dims               # device-less handle
    two = [nn.Sequential(nn.Linear(od, 32), nn.ReLU(), nn.Linear(32, 32), nn.ReLU(), nn.Linear(32, 5)) for od in obs_dims]
    one = [nn.Sequential(nn.Linear(od, 32), nn.ReLU(), nn.Linear(32, 5)) for od in obs_dims]
    for mode in ("argmax", "Categorical", None):
        with pytest.raises(ValueError, match="action_mode"):
            env.rollout_policy(two, 4, action_mode=mode)
    with pytest.raises(ValueError, match="record_log_probs"):
        env.rollout_policy(two, 4, record_log_probs=True)
    with pytest.raises(ValueError, match="record_log_probs"):
        env.rollout_policy(two, 4, action_mode="softmax", record_log_probs=True)
    with pytest.raises(NotImplementedError, match="two-hidden-layer"):
        env.rollout_policy(one, 4, action_mode="categorical")
    with pytest.raises(NotImplementedError, match="two-hidden-layer"):
        env.rollout_policy(one, 4, action_mode="categorical", record_log_probs=True)
