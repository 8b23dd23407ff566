"""env.rollout_policy with MADDPG's two-hidden-layer actor (mpe_rollout_policy_mlp: T steps in one launch, the actor
evaluated on the tensor cores in TF32): environment parity with ordinary fused steps, observation records, the actor's
numerics against float64, the Gumbel-softmax exploration stream, and the interface."""
import numpy as np
import pytest

from helpers import make_product_env
from mlp_helpers import actor_logits, explain_tf32_mismatches, gumbel_noise, softmax, tf32_tie

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

# Every (scenario, H) instantiation of mpe_policy_mlp_rollout_kernel at three launch shapes (helpers.launch_shape "mlp":
# ceil(warps / SMs) warps per block, capped at 16, or 12 for tag at H = 64):
#   "one"  a ragged size with 1-warp blocks
#   "mid"  5-warp blocks with a partial last block and a partial last warp
#   "full" 65 536 worlds plus a ragged tail: 16-warp blocks (12 for tag H = 64), partial last block and warp
# Explore settings: "one" and "mid" run both; "full" explores at H = 64 and runs the deterministic actor at H = 32.
CASES = [(tag, shape, T, H) for tag, T0 in (("simple_spread_n3", 12), ("simple_tag", 10), ("simple", 6))
         for H in (32, 64) for shape, T in (("one", T0), ("mid", 4), ("full", 2))]
MLP_PARAMS = [c + (e,) for c in CASES for e in ((False, True) if c[1] != "full" else (c[3] == 64,))]
MLP_SIZES = {"one": dict(wpb=1, base=2048), "mid": dict(wpb=5), "full": dict(wpb=16, base=65536)}

# Actor numerics, recorded actions vs float64 with the kernel's TF32 operand rounding: every row beyond 1e-5 must be
# a TF32 rounding flip (mlp_helpers.explain_tf32_mismatches); a few percent of rows are.
TIGHT_ATOL = 1e-5
# Loose: no rounding in the reference; TF32 keeps 11 significant bits (relative error <= 2^-11 per operand), which at
# these weight scales (unit-variance pre-activations) moves the probabilities by ~1e-3.  Bound 5e-3, 4.5x the observed.
LOOSE_MAX = 5e-3


def mlp_size(tag, shape, H):
    """the batch size of a CASES shape on this device, checked against the launch rule it is meant to exercise"""
    from helpers import device_sms, launch_shape, regime_size
    from mlp_programs import mlp_block_cap
    sms, cap = device_sms(), mlp_block_cap(tag, H)
    kw = dict(MLP_SIZES[shape])
    wpb = min(kw.pop("wpb"), cap)
    n = regime_size("mlp", sms, wpb, cap=cap, **kw)
    got = launch_shape("mlp", n, sms, cap)
    assert got[0] == wpb and got[2] == (wpb > 1) and got[3] < 32, (tag, shape, H, n, got)
    assert shape != "full" or (n > 65536 and wpb == cap)
    return n


def tf32_ties(W, every=3):
    """every `every`-th entry of W on a TF32 rounding tie, so that an actor which does not round ties away from zero,
    as cvt.rna does, differs in every row"""
    return torch.as_tensor(tf32_tie(W.cpu().numpy(), every), device=W.device)


def make_policies(obs_dims, H, seed=3):
    g = torch.Generator(device="cuda").manual_seed(seed)
    pols = []
    for od in obs_dims:
        r = lambda *s: torch.randn(*s, device="cuda", generator=g)   # noqa: E731
        pols.append((tf32_ties(r(H, od) * 1.5 / od ** 0.5), r(H) * 0.3, tf32_ties(r(H, H) * 1.5 / H ** 0.5), r(H) * 0.3,
                     tf32_ties(r(5, H) * 1.5 / H ** 0.5), r(5) * 0.2))
    return pols


def as_sequential(pols):
    mods = []
    for W1, b1, W2, b2, W3, b3 in pols:
        H = W1.shape[0]
        m = torch.nn.Sequential(torch.nn.Linear(W1.shape[1], H), torch.nn.ReLU(), torch.nn.Linear(H, H), torch.nn.ReLU(),
                                torch.nn.Linear(H, 5)).cuda()
        with torch.no_grad():
            for lin, W, b in ((m[0], W1, b1), (m[2], W2, b2), (m[4], W3, b3)):
                lin.weight.copy_(W)
                lin.bias.copy_(b)
        mods.append(m)
    return mods


def twin_envs(tag, n, seed=9, **kw):
    a = make_product_env(tag, num_envs=n, seed=seed, **kw)
    b = make_product_env(tag, num_envs=n, seed=seed, **kw)
    a.reset()
    obs_b = b.reset()
    assert torch.equal(a.world.native.agent_pv, b.world.native.agent_pv)
    return a, b, obs_b


@pytest.mark.parametrize("tag,shape,T,H,explore", MLP_PARAMS)
def test_mlp_rollout_parity_records_and_numerics(tag, shape, T, H, explore):
    """(1) the recorded actions fed to T fused steps of a twin env reproduce the final state, the final observations,
    every step's rewards and the reward sums bit for bit; (2) obs_record[i][t] is the twin's observation before step t,
    bit for bit; (3) every action matches the float64 actor (+ the NumPy Gumbel noise when exploring) to 1e-5 unless
    the row is a TF32 rounding flip, and the unrounded float64 actor to LOOSE_MAX."""
    n = mlp_size(tag, shape, H)
    env_a, env_b, obs_b = twin_envs(tag, n)
    na, nb = env_a.world.native, env_b.world.native
    pols = make_policies(na.obs_dims, H)
    seed = 0x1234_5678_9ABC if explore else None
    obs_r, rew_r, done_r, _, ex = env_a.rollout_policy(pols, T, record_actions=True, per_step_rewards=True,
                                                       record_observations=True, explore_seed=seed)
    acts, rew_steps, obs_rec = ex["actions"], ex["rewards"], ex["observations"]
    assert env_a.explore_epoch == (1 if explore else 0)
    pols_np = [[t.cpu().numpy() for t in p] for p in pols]
    A = env_a.n
    rew_sum = torch.zeros(A, n, device="cuda")
    flips, lmax = 0, 0.0
    for t in range(T):
        for i in range(A):
            assert torch.equal(obs_rec[i][t], obs_b[i]), (t, i)
            o = obs_b[i].cpu().numpy()
            g = gumbel_noise(seed, 0, np.arange(n), t, i, A) if explore else 0.0
            got = acts[i][t].cpu().numpy().astype(np.float64)
            flips += explain_tf32_mismatches(got, o, pols_np[i], noise=g, atol=TIGHT_ATOL)
            lmax = max(lmax, float(np.abs(got - softmax(actor_logits(o, *pols_np[i], tf32=False) + g)).max()))
        obs_b, rew_s, _, _ = env_b.step([a[t] for a in acts])
        rew_sum += torch.stack(list(rew_s))
        assert torch.equal(rew_steps[t], torch.stack(list(rew_s))), t
    torch.cuda.synchronize()
    assert torch.equal(na.agent_pv, nb.agent_pv)
    for x, y in zip(obs_r, obs_b):
        assert torch.equal(x, y)
    assert torch.equal(torch.stack(list(rew_r)), rew_sum)
    assert not any(bool(d.any()) for d in done_r)
    print("\nMLP actor numerics %s H=%d %s n=%d explore=%s: %d of %d rows explained by TF32 rounding flips, loose max "
          "%.3e" % (tag, H, shape, n, explore, flips, n * T * A, lmax))
    assert lmax <= LOOSE_MAX


def test_exploration_is_reproducible_and_advances():
    tag, n, T = "simple_spread_n3", 2049, 5
    env_a, env_b, _ = twin_envs(tag, n)
    pols = make_policies(env_a.world.native.obs_dims, 64)
    start_pv = env_a.world.native.agent_pv.clone()
    _, _, _, _, ex_a = env_a.rollout_policy(pols, T, record_actions=True, explore_seed=77)
    _, _, _, _, ex_b = env_b.rollout_policy(pols, T, record_actions=True, explore_seed=77)
    assert all(torch.equal(x, y) for x, y in zip(ex_a["actions"], ex_b["actions"]))
    assert torch.equal(env_a.world.native.agent_pv, env_b.world.native.agent_pv)
    # the next call from the same state draws fresh noise (epoch 1)
    env_a.world.native.agent_pv.copy_(start_pv)
    _, _, _, _, ex_c = env_a.rollout_policy(pols, T, record_actions=True, explore_seed=77)
    assert env_a.explore_epoch == 2
    assert not torch.equal(ex_c["actions"][0][0], ex_a["actions"][0][0])
    # ... and differs from the deterministic actor, which does not advance the epoch
    env_a.world.native.agent_pv.copy_(start_pv)
    _, _, _, _, ex_d = env_a.rollout_policy(pols, T, record_actions=True)
    assert env_a.explore_epoch == 2 and not torch.equal(ex_d["actions"][0][0], ex_a["actions"][0][0])


def test_exploration_samples_follow_softmax_of_fixed_logits():
    """W3 = 0, b3 = fixed logits: the arg-max of the Gumbel-softmax sample is a draw from softmax(b3).  Chi-square over
    65 536 worlds x 2 steps; the draws are fixed by the seed, so the verdict is too."""
    from scipy.stats import chisquare
    n, T, H = 65536, 2, 32
    env = make_product_env("simple", num_envs=n, seed=4)
    env.reset()
    b3 = torch.tensor([0.5, -0.3, 1.0, 0.0, -1.0], device="cuda")
    W1, b1, W2, b2, _, _ = make_policies(env.world.native.obs_dims, H)[0]
    pol = (W1, b1, W2, b2, torch.zeros(5, H, device="cuda"), b3)
    _, _, _, _, ex = env.rollout_policy([pol], T, record_actions=True, explore_seed=2024)
    k = ex["actions"][0].argmax(-1).reshape(-1).cpu().numpy()
    counts = np.bincount(k, minlength=5)
    expect = softmax(b3.cpu().numpy().astype(np.float64)) * k.size
    stat, p = chisquare(counts, expect)
    assert p > 1e-3, (counts, expect, p)


def test_exploration_is_independent_of_sharding():
    tag, n, T = "simple_tag", 1031, 4
    full = make_product_env(tag, num_envs=n, seed=9)
    full.reset()
    pols = make_policies(full.world.native.obs_dims, 64)
    _, _, _, _, ex = full.rollout_policy(pols, T, record_actions=True, explore_seed=31)
    lo = 0
    for rank in range(2):
        sh = make_product_env(tag, num_envs=n, seed=9, rank=rank, world_size=2)
        sh.reset()
        m = sh.world.native.n_env
        assert sh.world.native.world_offset == lo
        _, _, _, _, exs = sh.rollout_policy(pols, T, record_actions=True, explore_seed=31)
        for a, b in zip(exs["actions"], ex["actions"]):
            assert torch.equal(a, b[:, lo:lo + m])
        lo += m
    assert lo == n


def test_mlp_rollout_interface():
    from multiagent_particle_envs_b200._lib import MpeError
    tag, n, T = "simple_tag", 1031, 6
    env_a, env_b, _ = twin_envs(tag, n)
    pols = make_policies(env_a.world.native.obs_dims, 64)
    # nn.Sequential == 6-tuple, bit for bit; records do not change the result
    obs_a, rew_a, _, _, ex_a = env_a.rollout_policy(as_sequential(pols), T, record_actions=True, explore_seed=5)
    obs_b, rew_b, _, _, ex_b = env_b.rollout_policy(pols, T, record_actions=True, per_step_rewards=True,
                                                    record_observations=True, explore_seed=5)
    assert all(torch.equal(x, y) for x, y in zip(ex_a["actions"], ex_b["actions"]))
    assert torch.equal(env_a.world.native.agent_pv, env_b.world.native.agent_pv)
    assert all(torch.equal(x, y) for x, y in zip(obs_a, obs_b)) and torch.equal(torch.stack(rew_a), torch.stack(rew_b))
    env_c, _, _ = twin_envs(tag, n)
    obs_c, rew_c, _, _, ex_c = env_c.rollout_policy(pols, T, explore_seed=5)
    assert ex_c["actions"] is None and ex_c["observations"] is None and ex_c["rewards"] is None
    assert torch.equal(env_c.world.native.agent_pv, env_a.world.native.agent_pv)
    assert all(torch.equal(x, y) for x, y in zip(obs_c, obs_a)) and torch.equal(torch.stack(rew_c), torch.stack(rew_a))
    # a program without the policy kernels refuses in the library
    env_w = make_product_env("simple_world_comm", num_envs=64)
    env_w.reset()
    with pytest.raises(MpeError):
        env_w.rollout_policy(make_policies(env_w.world.native.obs_dims, 32), 2)
    # hidden widths other than 32 / 64 are not built
    with pytest.raises(MpeError):
        env_c.rollout_policy(make_policies(env_c.world.native.obs_dims, 48), 2)
    # exploration and observation records need the two-hidden-layer actor
    one = [(W1, b1, W3.new_zeros(5, W1.shape[0]), b3) for W1, b1, _, _, W3, b3 in pols]
    with pytest.raises(NotImplementedError):
        env_c.rollout_policy(one, 2, explore_seed=1)
    with pytest.raises(NotImplementedError):
        env_c.rollout_policy(one, 2, record_observations=True)
    with pytest.raises(ValueError):
        env_c.rollout_policy([p[:5] + (torch.zeros(4, device="cuda"),) for p in pols], 2)
