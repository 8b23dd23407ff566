"""env.rollout_policy(..., episode_length=L) with MADDPG's two-hidden-layer actor (mpe_rollout_policy_mlp_episodes): E =
n_steps / L whole episodes in one launch, every world reset inside the kernel after each episode.  The contract is bit
for bit the loop a trainer writes without it,

    for e in range(E):
        obs_e, rew_e, _, _, ex_e = env.rollout_policy(actors, L, ..., explore_seed=s)
        env.reset()

run on a twin env: records, final observations, returns, state, epochs.  Checked for every program the kernel is built
for, at both hidden widths, with and without exploration, at a ragged launch shape and (for four programs) at 65 536
worlds plus a tail at the block cap; then reseeding, sharding, the device epoch and the interface."""
import pytest

from helpers import device_sms, launch_shape, make_product_env, regime_size
from mlp_programs import PROGRAMS, as_sequential, make_policies, mlp_block_cap, state, twins

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

RECORDS = dict(record_actions=True, per_step_rewards=True, record_observations=True)


def assert_same_state(a, b):
    for x, y, name in zip(state(a), state(b), ("pv", "lm", "comm", "goal")):
        assert torch.equal(x, y), name
    assert a.world.native.epoch == b.world.native.epoch
    assert a.explore_epoch == b.explore_epoch


def run_loop(env, pols, E, L, seed, **records):
    """the reference: E single-episode calls, each followed by env.reset()"""
    acts, rews, obss, finals, rets = [], [], [], [], []
    for _ in range(E):
        obs_e, rew_e, _, _, ex = env.rollout_policy(pols, L, explore_seed=seed, **records)
        acts.append(ex["actions"])
        rews.append(ex["rewards"])
        obss.append(ex["observations"])
        finals.append(obs_e)
        rets.append(rew_e)
        obs = env.reset()
    A = env.n
    out = dict(obs=obs, final=[torch.stack([f[i] for f in finals]) for i in range(A)],
               returns=[torch.stack([r[i] for r in rets]) for i in range(A)])
    if records.get("record_actions"):
        out["actions"] = [torch.cat([a[i] for a in acts]) for i in range(A)]
    if records.get("per_step_rewards"):
        out["rewards"] = torch.cat(rews)
    if records.get("record_observations"):
        out["observations"] = [torch.cat([o[i] for o in obss]) for i in range(A)]
    return out


def assert_matches_loop(env_a, env_b, pols, E, L, seed):
    obs, ret, done, _, ex = env_a.rollout_policy(pols, E * L, episode_length=L, explore_seed=seed, **RECORDS)
    ref = run_loop(env_b, pols, E, L, seed, **RECORDS)
    torch.cuda.synchronize()
    for i in range(env_a.n):
        assert torch.equal(ex["actions"][i], ref["actions"][i]), ("actions", i)
        assert torch.equal(ex["observations"][i], ref["observations"][i]), ("observations", i)
        assert torch.equal(ex["final_observations"][i], ref["final"][i]), ("final observations", i)
        assert ret[i].shape == (E, env_a.world.native.n_env) and torch.equal(ret[i], ref["returns"][i]), ("returns", i)
        assert torch.equal(obs[i], ref["obs"][i]), ("post-reset observations", i)
        assert not bool(done[i].any())
    assert torch.equal(ex["rewards"], ref["rewards"])
    assert_same_state(env_a, env_b)


def mid_size(tag, H):
    """min(5, cap)-warp blocks of the episode kernel with a partial last block and a partial last warp"""
    cap = mlp_block_cap(tag, H, episodes=True)
    return regime_size("mlp", device_sms(), min(5, cap), cap=cap)


@pytest.mark.parametrize("tag", tuple(PROGRAMS))
@pytest.mark.parametrize("H", [32, 64])
@pytest.mark.parametrize("E,L,explore", [(1, 6, True), (3, 4, False), (3, 5, True)])
def test_episodes_equal_the_loop(tag, H, E, L, explore):
    env_a, env_b = twins(tag, mid_size(tag, H))
    nw = env_a.world.native
    pols = make_policies(nw.obs_dims, nw.act_dims, H)
    epoch = nw.epoch
    assert_matches_loop(env_a, env_b, pols, E, L, 21 if explore else None)
    assert nw.epoch == epoch + E and env_a.explore_epoch == (E if explore else 0)


@pytest.mark.parametrize("tag,H", [("simple_spread_n3", 64), ("simple_spread_n6", 64), ("simple_tag_6v2", 64),
                                   ("simple_reference", 64), ("simple_spread_n3", 32)])
def test_episodes_equal_the_loop_at_the_block_cap(tag, H):
    """65 536 worlds plus a ragged tail, in blocks at the episode kernel's cap with a partial last block and warp"""
    sms = device_sms()
    cap = mlp_block_cap(tag, H, episodes=True)
    n = regime_size("mlp", sms, cap, cap=cap, base=65536)
    assert launch_shape("mlp", n, sms, cap)[0] == cap and n > 65536
    env_a, env_b = twins(tag, n)
    nw = env_a.world.native
    pols = make_policies(nw.obs_dims, nw.act_dims, H)
    assert_matches_loop(env_a, env_b, pols, 2, 3, 5)


@pytest.mark.parametrize("tag", ["simple_spread_n3", "simple_speaker_listener", "simple_tag_6v2"])
def test_reseeding_reproduces_the_episodes(tag):
    """after reset(seed=s) an E-episode call leaves the state reset(seed=s) plus E env.reset() calls leaves, and a
    second reset(seed=s) replays every record"""
    E, L, s = 3, 4, 1234
    env_a, env_b = twins(tag, 1031)
    nw = env_a.world.native
    pols = make_policies(nw.obs_dims, nw.act_dims, 32)
    env_a.reset(seed=s)
    _, ret1, _, _, ex1 = env_a.rollout_policy(pols, E * L, episode_length=L, explore_seed=3, **RECORDS)
    env_b.reset(seed=s)
    for _ in range(E):
        env_b.reset()
    env_b.explore_epoch = E
    assert_same_state(env_a, env_b)
    env_a.reset(seed=s)
    env_a.explore_epoch = 0
    _, ret2, _, _, ex2 = env_a.rollout_policy(pols, E * L, episode_length=L, explore_seed=3, **RECORDS)
    torch.cuda.synchronize()
    assert torch.equal(ex1["rewards"], ex2["rewards"])
    for key in ("actions", "observations", "final_observations"):
        for x, y in zip(ex1[key], ex2[key]):
            assert torch.equal(x, y), key
    for x, y in zip(ret1, ret2):
        assert torch.equal(x, y)
    assert_same_state(env_a, env_b)


@pytest.mark.parametrize("tag", ["simple_spread_n3", "simple_reference"])
def test_sharded_episodes_equal_the_full_batch(tag):
    """the global world index keys both the reset draw and the exploration noise"""
    E, L, n = 2, 3, 1031
    full = make_product_env(tag, num_envs=n, seed=9)
    full.reset()
    nw = full.world.native
    pols = make_policies(nw.obs_dims, nw.act_dims, 32)
    _, ret, _, _, ex = full.rollout_policy(pols, E * L, episode_length=L, explore_seed=77, **RECORDS)
    want = state(full)
    lo = 0
    for rank in range(2):
        sh = make_product_env(tag, num_envs=n, seed=9, rank=rank, world_size=2)
        sh.reset()
        m = sh.world.native.n_env
        assert sh.world.native.world_offset == lo
        _, ret_s, _, _, ex_s = sh.rollout_policy(pols, E * L, episode_length=L, explore_seed=77, **RECORDS)
        torch.cuda.synchronize()
        assert torch.equal(ex_s["rewards"], ex["rewards"][:, :, lo:lo + m])
        for key in ("actions", "observations", "final_observations"):
            for x, y in zip(ex_s[key], ex[key]):
                assert torch.equal(x, y[:, lo:lo + m]), key
        for x, y in zip(ret_s, ret):
            assert torch.equal(x, y[:, lo:lo + m])
        for x, y in zip(state(sh), want):
            assert torch.equal(x, y[..., lo:lo + m, :] if x.dim() == 3 else y[:, lo:lo + m])
        lo += m
    assert lo == n


def test_device_epoch_is_read_before_and_written_after():
    """with the reset epoch in device memory (as after a GraphedRollout), the episode call resets from the device's
    epoch and leaves it where E resets would, so that a following env.reset() continues the sequence"""
    E, L = 3, 2
    env_a, env_b = twins("simple_spread_n3", 1031)
    nw_a = env_a.world.native
    pols = make_policies(nw_a.obs_dims, nw_a.act_dims, 32)
    epoch = nw_a.epoch
    dev = nw_a.enable_device_epoch()
    dev.add_(5)                               # what five graphed resets would have left on the device
    for _ in range(5):
        env_b.reset()
    env_a.rollout_policy(pols, E * L, episode_length=L)
    run_loop(env_b, pols, E, L, None)
    assert int(dev.item()) == nw_a.epoch == env_b.world.native.epoch == epoch + 5 + E
    env_a.reset()
    env_b.reset()
    assert_same_state(env_a, env_b)
    assert int(dev.item()) == nw_a.epoch


@pytest.mark.parametrize("tag", ["simple_spread_n3", "simple_crypto"])
def test_sequential_actors_equal_tuples(tag):
    env_a, env_b = twins(tag, 1031)
    nw = env_a.world.native
    pols = make_policies(nw.obs_dims, nw.act_dims, 64)
    ra = env_a.rollout_policy(pols, 6, episode_length=3, explore_seed=2, **RECORDS)
    rb = env_b.rollout_policy(as_sequential(pols), 6, episode_length=3, explore_seed=2, **RECORDS)
    torch.cuda.synchronize()
    for x, y in zip(ra[0] + ra[1], rb[0] + rb[1]):
        assert torch.equal(x, y)
    assert torch.equal(ra[4]["rewards"], rb[4]["rewards"])
    for key in ("actions", "observations", "final_observations"):
        for x, y in zip(ra[4][key], rb[4][key]):
            assert torch.equal(x, y), key
    assert_same_state(env_a, env_b)


def test_refusals_leave_state_and_epochs_unchanged():
    from multiagent_particle_envs_b200._lib import MpeError
    env = make_product_env("simple_spread_n3", num_envs=64, seed=9)
    env.reset()
    nw = env.world.native
    before, epoch = state(env), nw.epoch
    pols = make_policies(nw.obs_dims, nw.act_dims, 32)

    def unchanged():
        torch.cuda.synchronize()
        for x, y in zip(state(env), before):
            assert torch.equal(x, y)
        assert nw.epoch == epoch and env.explore_epoch == 0

    for n_steps, L in ((7, 2), (4, 0), (4, -1), (0, 2), (2, 4)):
        with pytest.raises(ValueError, match="episode_length"):
            env.rollout_policy(pols, n_steps, episode_length=L, explore_seed=1)
        unchanged()
    one_layer = [torch.nn.Sequential(torch.nn.Linear(od, 32), torch.nn.ReLU(), torch.nn.Linear(32, 5)).cuda()
                 for od in nw.obs_dims]
    with pytest.raises(NotImplementedError, match="episode_length"):
        env.rollout_policy(one_layer, 4, episode_length=2)
    unchanged()
    wc = make_product_env("simple_world_comm", num_envs=64, seed=9)   # a program without the kernel
    wc.reset()
    wnw = wc.world.native
    wbefore, wepoch = state(wc), wnw.epoch
    with pytest.raises(MpeError, match="no compiled"):
        wc.rollout_policy(make_policies(wnw.obs_dims, wnw.act_dims, 32), 4, episode_length=2, explore_seed=1)
    torch.cuda.synchronize()
    for x, y in zip(state(wc), wbefore):
        assert torch.equal(x, y)
    assert wnw.epoch == wepoch and wc.explore_epoch == 0


def test_exploring_episodes_refuse_a_counter_overflow_per_episode():
    """(t * 8 + i) * 2 + b, t < episode_length, must stay below the tag bit 2^30: tag 6+2 with episodes of 2^26 + 1 steps
    is refused before anything runs (no records requested, nothing of that size is allocated)"""
    from multiagent_particle_envs_b200._lib import MpeError
    env = make_product_env("simple_tag_6v2", num_envs=64, seed=9)
    env.reset()
    nw = env.world.native
    before, epoch = state(env), nw.epoch
    pols = make_policies(nw.obs_dims, nw.act_dims, 32)
    with pytest.raises(MpeError, match="bad argument"):
        env.rollout_policy(pols, 2 ** 26 + 1, episode_length=2 ** 26 + 1, explore_seed=1)
    torch.cuda.synchronize()
    for x, y in zip(state(env), before):
        assert torch.equal(x, y)
    assert nw.epoch == epoch and env.explore_epoch == 0


def test_records_are_none_unless_requested():
    env = make_product_env("simple_speaker_listener", num_envs=100, seed=9)
    env.reset()
    nw = env.world.native
    epoch = nw.epoch
    obs, ret, done, info, ex = env.rollout_policy(make_policies(nw.obs_dims, nw.act_dims, 32), 6, episode_length=2)
    assert ex == {"actions": None, "rewards": None, "observations": None, "final_observations": None}
    assert [r.shape for r in ret] == [(3, 100)] * env.n and [o.shape[0] for o in obs] == [100] * env.n
    assert nw.epoch == epoch + 3 and env.explore_epoch == 0
