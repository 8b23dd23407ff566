"""env.rollout_policy with MADDPG's two-hidden-layer actor (mpe_rollout_policy_mlp) on the scenarios with speaking or
immovable agents: simple_speaker_listener, simple_reference, simple_crypto, simple_adversary and simple_push.  The
actor's outputs split into the action sub-spaces (movement, utterance), each with its own (Gumbel-)softmax; an
utterance becomes the comm state after the step.  Checked: parity with ordinary fused steps fed with the recorded
actions (state, comm state, observations, rewards), the actor's numerics against float64 per sub-space, the exploration
stream, and the interface."""
import numpy as np
import pytest

from helpers import descriptor, make_product_env
from mlp_helpers import actor_logits, explain_tf32_mismatches, gumbel_noise, segment_softmax
from mlp_programs import LOOSE_MAX, TIGHT_ATOL, as_sequential, make_policies, mlp_block_cap

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

COMM_TAGS = ("simple_speaker_listener", "simple_reference", "simple_crypto", "simple_adversary", "simple_push")

# Every (scenario, H) instantiation at three launch shapes (helpers.launch_shape "mlp": ceil(warps / SMs) warps per
# block, capped at mlp_programs.mlp_block_cap -- 12 for simple_reference at H = 64, else 16):
#   "one"  a ragged size with 1-warp blocks
#   "mid"  5-warp blocks with a partial last block and a partial last warp
#   "full" 65 536 worlds plus a ragged tail at the full cap, partial last block and warp
# "one" and "mid" run with and without exploration; "full" explores at H = 64 and runs the deterministic actor at H = 32.
CASES = [(tag, shape, T, H) for tag in COMM_TAGS for H in (32, 64) for shape, T in (("one", 8), ("mid", 4), ("full", 2))]
MLP_PARAMS = [c + (e,) for c in CASES for e in ((False, True) if c[1] != "full" else (c[3] == 64,))]
MLP_SIZES = {"one": dict(wpb=1, base=2048), "mid": dict(wpb=5), "full": dict(wpb=16, base=65536)}

SEGMENT_SUM_ATOL = 2e-6


def segments(tag):
    """per agent, the widths of its action sub-spaces in action-vector order: [5] if movable, then [dim_c] if it speaks"""
    d = descriptor(tag)
    return [([5] if d.agent_movable[i] else []) + ([d.dim_c] if not d.agent_silent[i] else []) for i in range(d.n_agents)]


def explore_stride(act_dims):
    return 2 if max(act_dims) <= 8 else 4


def mlp_size(tag, shape, H):
    """the batch size of a CASES shape on this device, checked against the launch rule it is meant to exercise"""
    from helpers import device_sms, launch_shape, regime_size
    sms, cap = device_sms(), mlp_block_cap(tag, H)
    kw = dict(MLP_SIZES[shape])
    wpb = min(kw.pop("wpb"), cap)
    n = regime_size("mlp", sms, wpb, cap=cap, **kw)
    got = launch_shape("mlp", n, sms, cap)
    assert got[0] == wpb and got[2] == (wpb > 1) and got[3] < 32, (shape, H, n, got)
    assert shape != "one" or got[0] == 1
    assert shape != "full" or (n >= 65536 and wpb == cap)
    return n


def twin_envs(tag, n, seed=9, **kw):
    """two identical envs after reset, with a non-zero comm state (so that the rollout must load it), and the second
    one's observations of that state"""
    a = make_product_env(tag, num_envs=n, seed=seed, **kw)
    b = make_product_env(tag, num_envs=n, seed=seed, **kw)
    a.reset()
    b.reset()
    na, nb = a.world.native, b.world.native
    assert torch.equal(na.agent_pv, nb.agent_pv) and torch.equal(na.goal, nb.goal)
    if na.n_speakers > 0:
        g = torch.Generator(device="cuda").manual_seed(seed)
        c = torch.rand(na.comm.shape, device="cuda", generator=g)
        na.comm.copy_(c)
        nb.comm.copy_(c)
    obs_b = [o.clone() for o in nb.observe(out=nb.new_outputs(), flags=b._flags()).obs]
    return a, b, obs_b


@pytest.mark.parametrize("tag,shape,T,H,explore", MLP_PARAMS)
def test_comm_rollout_parity_records_and_numerics(tag, shape, T, H, explore):
    """(1) the recorded actions fed to T fused steps of a twin env reproduce the final state and comm state, the final
    observations, every step's rewards and the reward sums bit for bit, and immovable agents never move; (2)
    obs_record[i][t] is the twin's observation before step t, bit for bit; (3) every action matches the float64 actor
    (+ the NumPy Gumbel noise when exploring), one softmax per sub-space, to 1e-5 unless the row is a TF32 rounding
    flip, and the unrounded float64 actor to LOOSE_MAX; each sub-space sums to one."""
    shapes = make_product_env(tag, num_envs=1).world.native_shapes()
    A, act_dims, segs = shapes.n_agents, list(shapes.act_dims), segments(tag)
    assert [sum(s) for s in segs] == act_dims
    n = mlp_size(tag, shape, H)
    env_a, env_b, obs_b = twin_envs(tag, n)
    na, nb = env_a.world.native, env_b.world.native
    desc = descriptor(tag)
    pv0 = na.agent_pv.clone()
    pols = make_policies(na.obs_dims, act_dims, H)
    seed = 0x1234_5678_9ABC if explore else None
    obs_r, rew_r, done_r, _, ex = env_a.rollout_policy(pols, T, record_actions=True, per_step_rewards=True,
                                                       record_observations=True, explore_seed=seed)
    acts, rew_steps, obs_rec = ex["actions"], ex["rewards"], ex["observations"]
    assert [tuple(a.shape) for a in acts] == [(T, n, ad) for ad in act_dims]
    assert env_a.explore_epoch == (1 if explore else 0)
    pols_np = [[t.cpu().numpy() for t in p] for p in pols]
    stride = explore_stride(act_dims)
    rew_sum = torch.zeros(A, n, device="cuda")
    flips, lmax, smax = 0, 0.0, 0.0
    for t in range(T):
        for i in range(A):
            assert torch.equal(obs_rec[i][t], obs_b[i]), (t, i)
            o = obs_b[i].cpu().numpy()
            g = gumbel_noise(seed, 0, np.arange(n), t, i, A, n_logits=act_dims[i], stride=stride) if explore else 0.0
            got = acts[i][t].cpu().numpy().astype(np.float64)
            flips += explain_tf32_mismatches(got, o, pols_np[i], noise=g, atol=TIGHT_ATOL, segments=segs[i])
            want = segment_softmax(actor_logits(o, *pols_np[i], tf32=False) + g, segs[i])
            lmax = max(lmax, float(np.abs(got - want).max()))
            c = 0
            for w in segs[i]:
                smax = max(smax, float(np.abs(got[:, c:c + w].sum(-1) - 1.0).max()))
                c += w
        obs_b, rew_s, _, _ = env_b.step([a[t] for a in acts])
        rew_sum += torch.stack(list(rew_s))
        assert torch.equal(rew_steps[t], torch.stack(list(rew_s))), t
    torch.cuda.synchronize()
    assert torch.equal(na.agent_pv, nb.agent_pv)
    assert torch.equal(na.comm, nb.comm)
    for i in range(A):
        if not desc.agent_movable[i]:
            assert torch.equal(na.agent_pv[i], pv0[i]), i
    for x, y in zip(obs_r, obs_b):
        assert torch.equal(x, y)
    assert torch.equal(torch.stack(list(rew_r)), rew_sum)
    assert not any(bool(d.any()) for d in done_r)
    print("\nMLP actor numerics %s H=%d %s n=%d explore=%s: %d of %d rows explained by TF32 rounding flips, loose max "
          "%.3e, segment sums within %.1e of 1" % (tag, H, shape, n, explore, flips, n * T * A, lmax, smax))
    assert lmax <= LOOSE_MAX
    assert smax <= SEGMENT_SUM_ATOL


def _fixed_logit_policies(env, H, b3_of):
    """agents' actors with W3 = 0 and b3 = b3_of(i) (None: the seeded actor)"""
    nw = env.world.native
    pols = make_policies(nw.obs_dims, nw.act_dims, H)
    out = []
    for i, (W1, b1, W2, b2, W3, b3) in enumerate(pols):
        fixed = b3_of(i)
        if fixed is not None:
            W3, b3 = torch.zeros_like(W3), torch.tensor(fixed, dtype=torch.float32, device="cuda")
        out.append((W1, b1, W2, b2, W3, b3))
    return out


def test_speaker_utterance_samples_follow_softmax_of_fixed_logits():
    """W3 = 0: the arg-max of the speaker's Gumbel-softmax utterance is a draw from softmax(b3).  Chi-square over
    65 536 worlds x 2 steps; the draws are fixed by the seed, so the verdict is too."""
    from scipy.stats import chisquare
    n, T = 65536, 2
    env = make_product_env("simple_speaker_listener", num_envs=n, seed=4)
    env.reset()
    b3 = [0.4, -0.6, 0.9]
    pols = _fixed_logit_policies(env, 32, lambda i: b3 if i == 0 else None)
    _, _, _, _, ex = env.rollout_policy(pols, T, record_actions=True, explore_seed=2024)
    k = ex["actions"][0].argmax(-1).reshape(-1).cpu().numpy()
    counts = np.bincount(k, minlength=3)
    expect = segment_softmax(np.asarray(b3, np.float64)) * k.size
    stat, p = chisquare(counts, expect)
    assert p > 1e-3, (counts, expect, p)


def test_reference_joint_movement_and_utterance_samples_are_independent_draws():
    """W3 = 0: agent 0 of simple_reference draws its movement from softmax(b3[:5]) and its utterance from
    softmax(b3[5:]), independently.  Chi-square over the 5 x 10 table of (movement arg-max, utterance arg-max): uniforms
    shared between the sub-spaces or between Philox blocks would couple the two."""
    from scipy.stats import chisquare
    n, T = 65536, 2
    env = make_product_env("simple_reference", num_envs=n, seed=4)
    env.reset()
    b3 = [0.5, -0.3, 1.0, 0.0, -1.0] + list(np.linspace(-0.6, 0.6, 10))
    pols = _fixed_logit_policies(env, 64, lambda i: b3 if i == 0 else None)
    _, _, _, _, ex = env.rollout_policy(pols, T, record_actions=True, explore_seed=2025)
    a = ex["actions"][0].reshape(-1, 15).cpu().numpy()
    k = a[:, :5].argmax(-1) * 10 + a[:, 5:].argmax(-1)
    counts = np.bincount(k, minlength=50)
    z = np.asarray(b3, np.float64)
    expect = np.outer(segment_softmax(z[:5]), segment_softmax(z[5:])).reshape(-1) * k.size
    assert expect.min() > 100
    stat, p = chisquare(counts, expect)
    assert p > 1e-3, (counts, expect, p)


@pytest.mark.parametrize("tag", ["simple_reference", "simple_crypto"])
def test_comm_exploration_is_reproducible_and_advances(tag):
    n, T = 2049, 5
    env_a, env_b, _ = twin_envs(tag, n)
    nw = env_a.world.native
    pols = make_policies(nw.obs_dims, nw.act_dims, 64)
    start_pv, start_c = nw.agent_pv.clone(), nw.comm.clone()
    _, _, _, _, ex_a = env_a.rollout_policy(pols, T, record_actions=True, explore_seed=77)
    _, _, _, _, ex_b = env_b.rollout_policy(pols, T, record_actions=True, explore_seed=77)
    assert all(torch.equal(x, y) for x, y in zip(ex_a["actions"], ex_b["actions"]))
    assert torch.equal(nw.agent_pv, env_b.world.native.agent_pv) and torch.equal(nw.comm, env_b.world.native.comm)
    # the next call from the same state draws fresh noise (epoch 1)
    nw.agent_pv.copy_(start_pv)
    nw.comm.copy_(start_c)
    _, _, _, _, ex_c = env_a.rollout_policy(pols, T, record_actions=True, explore_seed=77)
    assert env_a.explore_epoch == 2
    assert not torch.equal(ex_c["actions"][0][0], ex_a["actions"][0][0])
    # ... and differs from the deterministic actor, which does not advance the epoch
    nw.agent_pv.copy_(start_pv)
    nw.comm.copy_(start_c)
    _, _, _, _, ex_d = env_a.rollout_policy(pols, T, record_actions=True)
    assert env_a.explore_epoch == 2 and not torch.equal(ex_d["actions"][0][0], ex_a["actions"][0][0])


def test_reference_exploration_is_independent_of_sharding():
    tag, n, T = "simple_reference", 1031, 4
    full = make_product_env(tag, num_envs=n, seed=9)
    full.reset()
    nw = full.world.native
    pols = make_policies(nw.obs_dims, nw.act_dims, 64)
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


def test_reference_exploring_rollout_refuses_a_counter_overflow():
    """simple_reference draws 4 Philox blocks per agent and step: (t * 2 + i) * 4 + b must stay below the counter's tag
    bit 2^30, so 2^27 + 1 steps are refused before anything runs (no records requested, nothing of that size is
    allocated)"""
    from multiagent_particle_envs_b200._lib import MpeError
    env = make_product_env("simple_reference", num_envs=64, seed=9)
    env.reset()
    nw = env.world.native
    pv, c = nw.agent_pv.clone(), nw.comm.clone()
    pols = make_policies(nw.obs_dims, nw.act_dims, 32)
    with pytest.raises(MpeError, match="bad argument"):
        env.rollout_policy(pols, 2 ** 27 + 1, explore_seed=1)
    torch.cuda.synchronize()
    assert env.explore_epoch == 0 and torch.equal(nw.agent_pv, pv) and torch.equal(nw.comm, c)


@pytest.mark.parametrize("tag", COMM_TAGS)
@pytest.mark.parametrize("H", [32, 64])
def test_comm_rollout_interface(tag, H):
    from multiagent_particle_envs_b200._lib import MpeError
    n, T = 1031, 5
    env_a, env_b, _ = twin_envs(tag, n)
    nw = env_a.world.native
    act_dims = list(nw.act_dims)
    pols = make_policies(nw.obs_dims, act_dims, H)
    # nn.Sequential == 6-tuple, bit for bit; records do not change the result
    obs_a, rew_a, _, _, ex_a = env_a.rollout_policy(as_sequential(pols), T, record_actions=True, explore_seed=5)
    obs_b, rew_b, _, _, ex_b = env_b.rollout_policy(pols, T, record_actions=True, per_step_rewards=True,
                                                    record_observations=True, explore_seed=5)
    assert [tuple(a.shape) for a in ex_a["actions"]] == [(T, n, ad) for ad in act_dims]
    assert all(torch.equal(x, y) for x, y in zip(ex_a["actions"], ex_b["actions"]))
    assert torch.equal(nw.agent_pv, env_b.world.native.agent_pv) and torch.equal(nw.comm, env_b.world.native.comm)
    assert all(torch.equal(x, y) for x, y in zip(obs_a, obs_b)) and torch.equal(torch.stack(rew_a), torch.stack(rew_b))
    env_c, _, _ = twin_envs(tag, n)
    obs_c, rew_c, _, _, ex_c = env_c.rollout_policy(pols, T, explore_seed=5)
    assert ex_c["actions"] is None and ex_c["observations"] is None and ex_c["rewards"] is None
    assert torch.equal(env_c.world.native.agent_pv, nw.agent_pv) and torch.equal(env_c.world.native.comm, nw.comm)
    assert all(torch.equal(x, y) for x, y in zip(obs_c, obs_a)) and torch.equal(torch.stack(rew_c), torch.stack(rew_a))
    # a head of the wrong width is refused before anything runs
    with pytest.raises(ValueError, match="W3 \\[%d, %d\\]" % (act_dims[0], H)):
        env_c.rollout_policy([p[:4] + (p[4].new_zeros(act_dims[0] + 1, H), p[5].new_zeros(act_dims[0] + 1))
                              if i == 0 else p for i, p in enumerate(pols)], 2)
    # the one-hidden-layer kernel is not built for these scenarios
    one = [(W1, b1, W3.new_zeros(5, H), b3.new_zeros(5)) for W1, b1, _, _, W3, b3 in pols]
    with pytest.raises(MpeError):
        env_c.rollout_policy(one, 2)


def test_world_comm_two_hidden_layer_actor_is_not_built():
    """simple_world_comm (six agents, observations of 28-34 floats) stays without the tensor-core actor"""
    from multiagent_particle_envs_b200._lib import MpeError
    env = make_product_env("simple_world_comm", num_envs=64)
    env.reset()
    nw = env.world.native
    with pytest.raises(MpeError):
        env.rollout_policy(make_policies(nw.obs_dims, nw.act_dims, 32), 2)
