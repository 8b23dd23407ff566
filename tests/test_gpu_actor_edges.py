"""Edge policies for the tensor-core actor (env.rollout_policy with a Linear-ReLU-Linear-ReLU-Linear policy,
mpe_rollout_policy_mlp): saturating logits, dead ReLUs, operands on exact TF32 ties, exploration at global world indices
beyond 2^32, and the refusal of an exploring rollout whose Philox counter would overflow."""
import numpy as np
import pytest

from helpers import make_product_env
from mlp_helpers import actor_logits, explain_tf32_mismatches, gumbel_noise, softmax, tf32_rna, tf32_rne, tf32_tie

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

N = 1031            # 33 warps: 1-warp blocks, ragged last warp


def _policy(obs_dim, H, seed, w3_scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda *s: torch.randn(*s, device="cuda", generator=g)   # noqa: E731
    return (r(H, obs_dim) * 1.5 / obs_dim ** 0.5, r(H) * 0.3, r(H, H) * 1.5 / H ** 0.5, r(H) * 0.3,
            r(5, H) * 1.5 / H ** 0.5 * w3_scale, r(5) * 0.2)


def _run(tag, pols, T, **kw):
    env = make_product_env(tag, num_envs=N, seed=9)
    env.reset()
    _, _, _, _, ex = env.rollout_policy(pols, T, record_actions=True, record_observations=True, **kw)
    torch.cuda.synchronize()
    return env, ex


@pytest.mark.parametrize("tag,H", [("simple_tag", 64), ("simple_spread_n3", 32)])
def test_saturating_logits_give_exact_one_hots(tag, H):
    """W3 scaled so that |logits| ~ 1e5: every action is an exact one-hot at the float64 arg-max, never NaN"""
    env = make_product_env(tag, num_envs=1)
    pols = [_policy(od, H, 10 + i, w3_scale=1e5) for i, od in enumerate(env.world.native.obs_dims)]
    env, ex = _run(tag, pols, 3)
    pols_np = [[t.cpu().numpy() for t in p] for p in pols]
    for i in range(env.n):
        for t in range(3):
            got = ex["actions"][i][t].cpu().numpy()
            assert np.isfinite(got).all()
            z = actor_logits(ex["observations"][i][t].cpu().numpy(), *pols_np[i])
            assert np.median(np.abs(z)) > 1e3
            top2 = np.sort(z, -1)[:, -2:]
            clear = top2[:, 1] - top2[:, 0] > 200.0          # every other expf underflows to exactly 0 in fp32
            assert clear.mean() > 0.99, clear.mean()
            one_hot = np.eye(5, dtype=np.float32)[z.argmax(-1)]
            assert np.array_equal(got[clear], one_hot[clear]), (i, t)
            assert np.allclose(got.sum(-1), 1.0, atol=1e-6)


def test_dead_relus_give_the_bias_policy_in_every_world():
    """b1 = -1e4: h1 = 0 everywhere, so every world's action is softmax(W3 relu(b2) + b3), bit for bit the same"""
    tag, H = "simple_spread_n3", 64
    env = make_product_env(tag, num_envs=1)
    pols = []
    for i, od in enumerate(env.world.native.obs_dims):
        W1, b1, W2, b2, W3, b3 = _policy(od, H, 20 + i)
        pols.append((W1, torch.full_like(b1, -1e4), W2, b2, W3, b3))
    env, ex = _run(tag, pols, 4)
    for i, (W1, b1, W2, b2, W3, b3) in enumerate(pols):
        acts = ex["actions"][i]
        assert torch.equal(acts, acts[:1, :1].expand_as(acts)), i
        h2 = tf32_rna(np.maximum(b2.cpu().numpy(), 0)).astype(np.float64)
        want = softmax(h2 @ tf32_rna(W3.cpu().numpy()).astype(np.float64).T + b3.cpu().numpy().astype(np.float64))
        np.testing.assert_allclose(acts[0, 0].cpu().numpy(), want, rtol=0, atol=2e-7)


@pytest.mark.parametrize("H", [32, 64])
def test_tf32_ties_round_away_from_zero(H):
    """Observations (the velocity and the landmark position of `simple`, the agent at the origin) and weights on exact
    TF32 ties.  W1 and W2 have one non-zero per row and zero biases, so every hidden unit is a single exact product and
    no accumulation error can move it: the kernel must match the ties-away model with no row left to explain, while
    nearest-even rounding would move the actions by > 1e-4."""
    rng = np.random.RandomState(H)
    tag = "simple"
    env = make_product_env(tag, num_envs=N, seed=9)
    env.reset()
    nw = env.world.native
    od = nw.obs_dims[0]
    mag = lambda *s: tf32_tie(rng.uniform(0.4, 1.8, s) * rng.choice([-1.0, 1.0], s))   # noqa: E731
    vel, lm = mag(N, 2), mag(N, 2)
    nw.agent_pv[0, :, 0:2] = 0.0
    nw.agent_pv[0, :, 2:4] = torch.as_tensor(vel, device="cuda")
    nw.lm_p[0] = torch.as_tensor(lm, device="cuda")
    W1 = np.zeros((H, od), np.float32)
    W1[np.arange(H), np.arange(H) % od] = mag(H)
    W2 = np.zeros((H, H), np.float32)
    W2[np.arange(H), rng.permutation(H)] = mag(H)
    W3 = mag(5, H) / np.float32(4)
    b3 = rng.randn(5).astype(np.float32)
    params = [W1, np.zeros(H, np.float32), W2, np.zeros(H, np.float32), W3, b3]
    pols = [tuple(torch.as_tensor(p, device="cuda") for p in params)]
    _, _, _, _, ex = env.rollout_policy(pols, 1, record_actions=True, record_observations=True)
    torch.cuda.synchronize()
    obs = ex["observations"][0][0].cpu().numpy()
    assert np.array_equal(obs, np.concatenate([vel, lm], 1))
    got = ex["actions"][0][0].cpu().numpy().astype(np.float64)
    want = softmax(actor_logits(obs, *params))
    assert explain_tf32_mismatches(got, obs, params, atol=1e-6) == 0
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-6)
    f64 = np.float64
    h1 = tf32_rne(np.maximum(tf32_rne(obs).astype(f64) @ tf32_rne(W1).astype(f64).T, 0).astype(np.float32))
    h2 = tf32_rne(np.maximum(h1.astype(f64) @ tf32_rne(W2).astype(f64).T, 0).astype(np.float32))
    rne = softmax(h2.astype(f64) @ tf32_rne(W3).astype(f64).T + b3)
    assert np.abs(rne - want).max() > 1e-4


def test_exploration_beyond_two_to_the_32_worlds():
    """world_offset = 2^32 + 5: the Philox counter's high word is 1, and the noise must be the model's at those global
    indices"""
    tag, H, T, seed = "simple_tag", 32, 3, 0xDEAD_BEEF_0123
    env = make_product_env(tag, num_envs=N, seed=9)
    env.reset()
    offset = 2 ** 32 + 5
    env.world.native.world_offset = offset
    pols = [_policy(od, H, 30 + i) for i, od in enumerate(env.world.native.obs_dims)]
    _, _, _, _, ex = env.rollout_policy(pols, T, record_actions=True, record_observations=True, explore_seed=seed)
    torch.cuda.synchronize()
    pols_np = [[t.cpu().numpy() for t in p] for p in pols]
    A, flips = env.n, 0
    for t in range(T):
        for i in range(A):
            g = gumbel_noise(seed, 0, offset + np.arange(N, dtype=np.uint64), t, i, A)
            assert not np.array_equal(g, gumbel_noise(seed, 0, 5 + np.arange(N, dtype=np.uint64), t, i, A))
            flips += explain_tf32_mismatches(ex["actions"][i][t].cpu().numpy(), ex["observations"][i][t].cpu().numpy(),
                                             pols_np[i], noise=g)
    print("\nexploration at world_offset 2^32 + 5: %d of %d rows explained by TF32 rounding flips" % (flips, N * T * A))


def test_exploring_rollout_refuses_a_counter_overflow():
    """(t * A + i) * 2 + b must stay below the counter's tag bit 2^30: with one agent, 2^29 + 1 steps are refused before
    anything runs (no records requested, so nothing of that size is allocated)"""
    from multiagent_particle_envs_b200._lib import MpeError
    env = make_product_env("simple", num_envs=64, seed=9)
    env.reset()
    pv = env.world.native.agent_pv.clone()
    pols = [_policy(env.world.native.obs_dims[0], 32, 40)]
    with pytest.raises(MpeError, match="bad argument"):
        env.rollout_policy(pols, 2 ** 29 + 1, explore_seed=1)
    torch.cuda.synchronize()
    assert env.explore_epoch == 0 and torch.equal(env.world.native.agent_pv, pv)
