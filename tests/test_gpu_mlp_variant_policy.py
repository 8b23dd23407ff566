"""env.rollout_policy with MADDPG's two-hidden-layer actor (mpe_rollout_policy_mlp) on the entity-count variants:
simple_spread N = 2, 4, 5, 6, simple_tag 1+1, 2+1, 4+2, 6+2 and simple_adversary with 4 agents.  Their weights fill up
to 212 KB of shared memory, so the block size is capped by shared memory as well as by registers.  Checked: parity with
ordinary fused steps fed with the recorded actions, the actor's numerics against float64, the launched block size
against the cap mirror, the exploration stream, and the interface."""
import json

import numpy as np
import pytest

from helpers import device_sms, launch_shape, make_product_env, regime_size
from mlp_helpers import actor_logits, explain_tf32_mismatches, gumbel_noise, softmax
from mlp_programs import LOOSE_MAX, TIGHT_ATOL, as_sequential, make_policies, mlp_block_cap
from mlp_programs import VARIANT_PROGRAMS as PROGRAMS

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

TAGS = tuple(PROGRAMS)
# Every (program, H) at the launch shapes of test_gpu_mlp_comm_policy.py, with the cap of mlp_block_cap:
#   "one"  a ragged size with 1-warp blocks
#   "mid"  min(5, cap)-warp blocks with a partial last block and a partial last warp
#   "full" 65 536 worlds plus a ragged tail at the cap, partial last block and warp
# "one" and "mid" run with and without exploration; "full" explores at H = 64 and runs the deterministic actor at H = 32.
CASES = [(tag, shape, T, H) for tag in TAGS for H in (32, 64) for shape, T in (("one", 8), ("mid", 4), ("full", 2))]
MLP_PARAMS = [c + (e,) for c in CASES for e in ((False, True) if c[1] != "full" else (c[3] == 64,))]
MLP_SIZES = {"one": dict(wpb=1, base=2048), "mid": dict(wpb=5), "full": dict(wpb=16, base=65536)}


def mlp_size(tag, shape, H):
    """the batch size of a CASES shape on this device, checked against the launch rule it is meant to exercise"""
    sms, cap = device_sms(), mlp_block_cap(tag, H)
    kw = dict(MLP_SIZES[shape])
    wpb = min(kw.pop("wpb"), cap)
    n = regime_size("mlp", sms, wpb, cap=cap, **kw)
    got = launch_shape("mlp", n, sms, cap)
    assert got[0] == wpb and got[2] == (wpb > 1) and got[3] < 32, (tag, shape, H, n, got)
    assert shape != "one" or got[0] == 1
    assert shape != "full" or (n >= 65536 and wpb == cap)
    return n


def twin_envs(tag, n, seed=9, **kw):
    a = make_product_env(tag, num_envs=n, seed=seed, **kw)
    b = make_product_env(tag, num_envs=n, seed=seed, **kw)
    a.reset()
    obs_b = b.reset()
    assert torch.equal(a.world.native.agent_pv, b.world.native.agent_pv)
    return a, b, obs_b


@pytest.mark.parametrize("tag,shape,T,H,explore", MLP_PARAMS)
def test_variant_rollout_parity_records_and_numerics(tag, shape, T, H, explore):
    """(1) the recorded actions fed to T fused steps of a twin env reproduce the final state, the final observations,
    every step's rewards and the reward sums bit for bit; (2) obs_record[i][t] is the twin's observation before step t,
    bit for bit; (3) every action matches the float64 actor (+ the NumPy Gumbel noise when exploring) to 1e-5 unless
    the row is a TF32 rounding flip, and the unrounded float64 actor to LOOSE_MAX."""
    n = mlp_size(tag, shape, H)
    env_a, env_b, obs_b = twin_envs(tag, n)
    na, nb = env_a.world.native, env_b.world.native
    A, act_dims = env_a.n, list(na.act_dims)
    assert act_dims == [5] * A
    pols = make_policies(na.obs_dims, act_dims, H)
    seed = 0x1234_5678_9ABC if explore else None
    obs_r, rew_r, done_r, _, ex = env_a.rollout_policy(pols, T, record_actions=True, per_step_rewards=True,
                                                       record_observations=True, explore_seed=seed)
    acts, rew_steps, obs_rec = ex["actions"], ex["rewards"], ex["observations"]
    assert env_a.explore_epoch == (1 if explore else 0)
    pols_np = [[t.cpu().numpy() for t in p] for p in pols]
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


@pytest.mark.parametrize("tag", TAGS)
@pytest.mark.parametrize("H", [32, 64])
def test_launched_block_size_is_the_mirrored_cap(tag, H, tmp_path):
    """the kernel's block and grid at the "full" size, read from a CUDA trace of the launch, are mlp_block_cap's: the
    mirror the other tests size their batches with is checked against the library, not against itself"""
    from torch.profiler import ProfilerActivity, profile
    n = mlp_size(tag, "full", H)
    cap = mlp_block_cap(tag, H)
    env = make_product_env(tag, num_envs=n, seed=9)
    env.reset()
    nw = env.world.native
    pols = make_policies(nw.obs_dims, nw.act_dims, H)
    env.rollout_policy(pols, 1)                                   # module load and attributes outside the trace
    torch.cuda.synchronize()
    # three launches: the trace may miss a kernel record (activity buffers are flushed asynchronously); every record
    # that is there must show the mirrored shape
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            env.rollout_policy(pols, 1)
        torch.cuda.synchronize()
    path = tmp_path / "trace.json"
    prof.export_chrome_trace(str(path))
    kernels = [e for e in json.loads(path.read_text())["traceEvents"] if e.get("cat") == "kernel"]
    events = [e for e in kernels if "mpe_policy_mlp_rollout_kernel" in e.get("name", "")]
    assert 1 <= len(events) <= 3, [e.get("name") for e in kernels]
    warps = -(-n // 32)
    for e in events:
        assert e["args"]["block"] == [32 * cap, 1, 1], (e["name"], e["args"])
        assert e["args"]["grid"] == [-(-warps // cap), 1, 1], (e["name"], e["args"])
        assert ", %d>" % H in e["name"], e["name"]


@pytest.mark.parametrize("tag", ["simple_spread_n6", "simple_tag_6v2"])
def test_variant_exploration_is_reproducible_advances_and_is_independent_of_sharding(tag):
    n, T = 2049, 5
    env_a, env_b, _ = twin_envs(tag, n)
    nw = env_a.world.native
    pols = make_policies(nw.obs_dims, nw.act_dims, 64)
    start_pv = nw.agent_pv.clone()
    _, _, _, _, ex_a = env_a.rollout_policy(pols, T, record_actions=True, explore_seed=77)
    _, _, _, _, ex_b = env_b.rollout_policy(pols, T, record_actions=True, explore_seed=77)
    assert all(torch.equal(x, y) for x, y in zip(ex_a["actions"], ex_b["actions"]))
    assert torch.equal(nw.agent_pv, env_b.world.native.agent_pv)
    # the next call from the same state draws fresh noise (epoch 1)
    nw.agent_pv.copy_(start_pv)
    _, _, _, _, ex_c = env_a.rollout_policy(pols, T, record_actions=True, explore_seed=77)
    assert env_a.explore_epoch == 2
    assert not torch.equal(ex_c["actions"][-1][0], ex_a["actions"][-1][0])
    # ... and differs from the deterministic actor, which does not advance the epoch
    nw.agent_pv.copy_(start_pv)
    _, _, _, _, ex_d = env_a.rollout_policy(pols, T, record_actions=True)
    assert env_a.explore_epoch == 2 and not torch.equal(ex_d["actions"][-1][0], ex_a["actions"][-1][0])
    # two shards draw the rows of the whole batch, bit for bit
    lo = 0
    for rank in range(2):
        sh = make_product_env(tag, num_envs=n, seed=9, rank=rank, world_size=2)
        sh.reset()
        m = sh.world.native.n_env
        assert sh.world.native.world_offset == lo
        _, _, _, _, exs = sh.rollout_policy(pols, T, record_actions=True, explore_seed=77)
        for a, b in zip(exs["actions"], ex_a["actions"]):
            assert torch.equal(a, b[:, lo:lo + m])
        lo += m
    assert lo == n


def test_tag_6v2_exploring_rollout_refuses_a_counter_overflow():
    """eight agents draw 2 Philox blocks each per step: (t * 8 + i) * 2 + b must stay below the counter's tag bit
    2^30, so 2^26 + 1 steps are refused before anything runs (no records requested, nothing of that size is
    allocated)"""
    from multiagent_particle_envs_b200._lib import MpeError
    env = make_product_env("simple_tag_6v2", num_envs=64, seed=9)
    env.reset()
    nw = env.world.native
    pv = nw.agent_pv.clone()
    pols = make_policies(nw.obs_dims, nw.act_dims, 32)
    with pytest.raises(MpeError, match="bad argument"):
        env.rollout_policy(pols, 2 ** 26 + 1, explore_seed=1)
    torch.cuda.synchronize()
    assert env.explore_epoch == 0 and torch.equal(nw.agent_pv, pv)


@pytest.mark.parametrize("tag", TAGS)
@pytest.mark.parametrize("H", [32, 64])
def test_variant_rollout_interface(tag, H):
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
    assert [tuple(a.shape) for a in ex_a["actions"]] == [(T, n, 5)] * len(act_dims)
    assert all(torch.equal(x, y) for x, y in zip(ex_a["actions"], ex_b["actions"]))
    assert torch.equal(nw.agent_pv, env_b.world.native.agent_pv)
    assert all(torch.equal(x, y) for x, y in zip(obs_a, obs_b)) and torch.equal(torch.stack(rew_a), torch.stack(rew_b))
    env_c, _, _ = twin_envs(tag, n)
    obs_c, rew_c, _, _, ex_c = env_c.rollout_policy(pols, T, explore_seed=5)
    assert ex_c["actions"] is None and ex_c["observations"] is None and ex_c["rewards"] is None
    assert torch.equal(env_c.world.native.agent_pv, nw.agent_pv)
    assert all(torch.equal(x, y) for x, y in zip(obs_c, obs_a)) and torch.equal(torch.stack(rew_c), torch.stack(rew_a))
    # a head of the wrong width is refused before anything runs
    with pytest.raises(ValueError, match="W3 \\[5, %d\\]" % H):
        env_c.rollout_policy([p[:4] + (p[4].new_zeros(6, H), p[5].new_zeros(6)) if i == 0 else p
                              for i, p in enumerate(pols)], 2)
    # the one-hidden-layer kernel is not built for these programs
    one = [(W1, b1, W3.new_zeros(5, H), b3.new_zeros(5)) for W1, b1, _, _, W3, b3 in pols]
    with pytest.raises(MpeError):
        env_c.rollout_policy(one, 2)
