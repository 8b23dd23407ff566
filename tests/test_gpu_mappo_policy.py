"""env.rollout_policy(..., action_mode="categorical") with MAPPO's actor (mpe_rollout_policy_mappo and its episode
form): [LayerNorm] -> Linear -> ReLU/Tanh -> LayerNorm -> Linear -> ReLU/Tanh -> LayerNorm -> Linear, H = 64.  Checked
for every program the kernel is built for, with ReLU and tanh, exploring and greedy, the input LayerNorm on for half of
the cases: replay of the recorded indices as one-hot vectors through fused steps of a twin env, bit for bit; every pick
and log-probability against the float64 model of the kernel's recipe and against the user's unfolded module; the
episode form against its loop; a shared policy module; the refusals."""
import numpy as np
import pytest

from helpers import device_sms, launch_shape, make_product_env, regime_size
from mappo_helpers import FEATURE_NORM, TANH, MappoModel, explain_mappo_mismatches, make_mappo_actors, module_logits
from mlp_categorical_helpers import bounds, log_softmax_at, one_hot_torch
from mlp_helpers import gumbel_noise
from mlp_programs import PROGRAMS, mlp_block_cap, state, twins

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

# the slack of tests/test_gpu_mlp_categorical.py: what a rounding flip adds to 2 max |dz| per sub-space
LOGP_FLIP_SLACK = 1e-3
RECORDS = dict(record_actions=True, per_step_rewards=True, record_observations=True, record_log_probs=True)


def segments_of(env):
    d = env.world.native.desc
    return [([5] if d.agent_movable[i] else []) + ([d.dim_c] if not d.agent_silent[i] else []) for i in range(env.n)]


def size(tag, wpb, base=None, episodes=False):
    cap = mlp_block_cap(tag, 64, episodes, categorical=True, mappo=True)
    sms = device_sms()
    n = regime_size("mlp", sms, min(wpb, cap), cap=cap, base=base)
    assert launch_shape("mlp", n, sms, cap)[0] == min(wpb, cap)
    return n


def observe(env):
    nw = env.world.native
    return [o.clone() for o in nw.observe(out=nw.new_outputs(), flags=env._flags()).obs]


def models_of(pols, nw):
    from multiagent_particle_envs_b200.environment import mappo_actor_params
    params, tanh, fn, eps = mappo_actor_params(pols, nw.obs_dims, nw.act_dims)
    net = ((FEATURE_NORM if fn else 0) | (TANH if tanh else 0), eps)
    return [MappoModel([t.to(torch.float32).cpu().numpy() for t in p], net) for p in params]


def check_replay_and_numerics(tag, n, T, explore, tanh, fn):
    env_a, env_b = twins(tag, n)
    na, nb = env_a.world.native, env_b.world.native
    A, act_dims, segs = env_a.n, list(na.act_dims), segments_of(env_a)
    pv0 = na.agent_pv.clone()
    pols = make_mappo_actors(na.obs_dims, act_dims, tanh, fn)
    models = models_of(pols, na)
    seed = 0x1234_5678_9ABC if explore else None
    obs_b = observe(env_b)
    obs_r, rew_r, done_r, _, ex = env_a.rollout_policy(pols, T, explore_seed=seed, action_mode="categorical", **RECORDS)
    idx, logp, rew_steps, obs_rec = ex["actions"], ex["log_probs"], ex["rewards"], ex["observations"]
    assert [(tuple(k.shape), k.dtype) for k in idx] == [((T, n, len(s)), torch.int32) for s in segs]
    assert tuple(logp.shape) == (T, A, n) and logp.dtype == torch.float32
    assert env_a.explore_epoch == (1 if explore else 0)
    rew_sum = torch.zeros(A, n, device="cuda")
    flips = gaps = 0
    lmax = 0.0
    stride = 2 if max(act_dims) <= 8 else 4
    for t in range(T):
        for i in range(A):
            assert torch.equal(obs_rec[i][t], obs_b[i]), (t, i)          # the raw observation
            o = obs_b[i].cpu().numpy()
            g = gumbel_noise(seed, 0, np.arange(n), t, i, A, n_logits=act_dims[i], stride=stride) if explore else 0.0
            k = idx[i][t].cpu().numpy()
            lp = logp[t, i].cpu().numpy().astype(np.float64)
            f, gp = explain_mappo_mismatches(k, lp, o, models[i], segs[i], noise=g)
            flips, gaps = flips + f, gaps + gp
            z64 = module_logits(pols[i], o)
            err = np.abs(lp - log_softmax_at(z64, k, segs[i]))
            lmax = max(lmax, float(err.max()))
            dz = np.abs(models[i](o) - z64)
            bound = sum(2.0 * dz[:, a:b].max(-1) for a, b in bounds(segs[i])) + LOGP_FLIP_SLACK
            assert (err <= bound).all(), (t, i, float((err - bound).max()))
        obs_b, rew_s, _, _ = env_b.step([one_hot_torch(k[t], s) for k, s in zip(idx, segs)])
        rew_sum += torch.stack(list(rew_s))
        assert torch.equal(rew_steps[t], torch.stack(list(rew_s))), t
    torch.cuda.synchronize()
    assert torch.equal(na.agent_pv, nb.agent_pv)
    assert torch.equal(na.comm, nb.comm)
    d = na.desc
    for i in range(A):
        if not d.agent_movable[i]:
            assert torch.equal(na.agent_pv[i], pv0[i]), i
    for x, y in zip(obs_r, obs_b):
        assert torch.equal(x, y)
    assert torch.equal(torch.stack(list(rew_r)), rew_sum)
    assert not any(bool(x.any()) for x in done_r)
    print("\nmappo %s tanh=%s feature_norm=%s n=%d explore=%s: %d of %d rows explained by TF32 rounding flips, %d by "
          "the Gumbel gap; log-probabilities within %.3e of the unfolded float64 module"
          % (tag, tanh, fn, n, explore, flips, n * T * A, gaps, lmax))


@pytest.mark.parametrize("tag", tuple(PROGRAMS))
@pytest.mark.parametrize("tanh", [False, True])
@pytest.mark.parametrize("explore", [True, False])
def test_mappo_replay_and_numerics(tag, tanh, explore):
    """a ragged multi-warp launch: min(5, cap)-warp blocks with a partial last block and a partial last warp; the input
    LayerNorm is on for (ReLU, exploring) and (tanh, greedy), so every program runs with and without it"""
    check_replay_and_numerics(tag, size(tag, 5), 3, explore, tanh, fn=(explore != tanh))


@pytest.mark.parametrize("tag,tanh,explore", [("simple_spread_n3", False, True), ("simple_reference", True, False),
                                              ("simple_tag_6v2", True, True)])
def test_mappo_replay_at_the_block_cap(tag, tanh, explore):
    """65 536 worlds plus a ragged tail in blocks at the kernel's cap"""
    check_replay_and_numerics(tag, size(tag, 16, base=65536), 2, explore, tanh, fn=True)


def mappo_loop(env, pols, E, L, seed):
    keys = ("actions", "rewards", "observations", "log_probs")
    parts = {k: [] for k in keys}
    finals, rets = [], []
    for _ in range(E):
        obs_e, rew_e, _, _, ex = env.rollout_policy(pols, L, explore_seed=seed, action_mode="categorical", **RECORDS)
        for k in keys:
            parts[k].append(ex[k])
        finals.append(obs_e)
        rets.append(rew_e)
        obs = env.reset()
    A = env.n
    return dict(obs=obs, final=[torch.stack([f[i] for f in finals]) for i in range(A)],
                returns=[torch.stack([r[i] for r in rets]) for i in range(A)],
                actions=[torch.cat([a[i] for a in parts["actions"]]) for i in range(A)],
                observations=[torch.cat([o[i] for o in parts["observations"]]) for i in range(A)],
                rewards=torch.cat(parts["rewards"]), log_probs=torch.cat(parts["log_probs"]))


@pytest.mark.parametrize("tag", tuple(PROGRAMS))
@pytest.mark.parametrize("E,L,explore,tanh,fn", [(3, 4, True, True, True), (2, 3, False, False, False)])
def test_mappo_episodes_equal_the_loop(tag, E, L, explore, tanh, fn):
    n = size(tag, 5, episodes=True)
    env_a, env_b = twins(tag, n)
    nw = env_a.world.native
    pols = make_mappo_actors(nw.obs_dims, nw.act_dims, tanh, fn)
    seed = 21 if explore else None
    epoch = nw.epoch
    obs, ret, done, _, ex = env_a.rollout_policy(pols, E * L, episode_length=L, explore_seed=seed,
                                                 action_mode="categorical", **RECORDS)
    ref = mappo_loop(env_b, pols, E, L, seed)
    torch.cuda.synchronize()
    for i in range(env_a.n):
        assert torch.equal(ex["actions"][i], ref["actions"][i]), ("actions", i)
        assert torch.equal(ex["observations"][i], ref["observations"][i]), ("observations", i)
        assert torch.equal(ex["final_observations"][i], ref["final"][i]), ("final observations", i)
        assert torch.equal(ret[i], ref["returns"][i]), ("returns", i)
        assert torch.equal(obs[i], ref["obs"][i]), ("post-reset observations", i)
        assert not bool(done[i].any())
    assert torch.equal(ex["rewards"], ref["rewards"])
    assert torch.equal(ex["log_probs"], ref["log_probs"])
    for x, y in zip(state(env_a), state(env_b)):
        assert torch.equal(x, y)
    assert nw.epoch == env_b.world.native.epoch == epoch + E
    assert env_a.explore_epoch == env_b.explore_epoch == (E if explore else 0)


def test_a_shared_policy_equals_equal_copies():
    """MAPPO's share_policy: one module object for the three agents of simple_spread N=3"""
    import copy
    env_a, env_b = twins("simple_spread_n3", 1031)
    nw = env_a.world.native
    shared = make_mappo_actors(nw.obs_dims[:1], nw.act_dims[:1], True, True)[0]
    ra = env_a.rollout_policy([shared] * 3, 5, explore_seed=2, action_mode="categorical", **RECORDS)
    rb = env_b.rollout_policy([copy.deepcopy(shared) for _ in range(3)], 5, explore_seed=2, action_mode="categorical",
                              **RECORDS)
    torch.cuda.synchronize()
    for x, y in zip(ra[0] + ra[1], rb[0] + rb[1]):
        assert torch.equal(x, y)
    for key in ("rewards", "log_probs"):
        assert torch.equal(ra[4][key], rb[4][key]), key
    for key in ("actions", "observations"):
        for x, y in zip(ra[4][key], rb[4][key]):
            assert torch.equal(x, y), key
    for x, y in zip(state(env_a), state(env_b)):
        assert torch.equal(x, y)


def test_refusals_leave_state_and_epochs_unchanged():
    from multiagent_particle_envs_b200 import _lib
    from multiagent_particle_envs_b200._lib import MpeError
    env = make_product_env("simple_spread_n3", num_envs=64, seed=9)
    env.reset()
    nw = env.world.native
    before, epoch = state(env), nw.epoch
    pols = make_mappo_actors(nw.obs_dims, nw.act_dims, False, True)

    def unchanged(e, b, ep):
        torch.cuda.synchronize()
        for x, y in zip(state(e), b):
            assert torch.equal(x, y)
        assert e.world.native.epoch == ep and e.explore_epoch == 0

    with pytest.raises(NotImplementedError, match="categorical"):
        env.rollout_policy(pols, 4, explore_seed=1)
    unchanged(env, before, epoch)
    with pytest.raises(NotImplementedError, match="hidden width 64"):
        env.rollout_policy(make_mappo_actors(nw.obs_dims, nw.act_dims, False, True, hidden=32), 4,
                           action_mode="categorical")
    unchanged(env, before, epoch)
    env.discrete_action_input = True
    with pytest.raises(NotImplementedError, match="plain action vectors"):
        env.rollout_policy(pols, 4, action_mode="categorical")
    env.discrete_action_input = False
    unchanged(env, before, epoch)
    # the library refuses H = 32 and unknown network flags itself
    from multiagent_particle_envs_b200.environment import mappo_actor_params
    params = mappo_actor_params(pols, nw.obs_dims, nw.act_dims)[0]
    keep = [[t.to(torch.float32).contiguous() for t in p] for p in params]
    w_ptrs = [_lib.ptr_array([keep[i][j].data_ptr() for i in range(3)]) for j in range(6)]
    with pytest.raises(MpeError, match="unsupported|not supported|no compiled"):
        nw.rollout_policy_mlp(w_ptrs, 32, 4, categorical=True, mappo=(0, 1e-5))
    with pytest.raises(MpeError, match="bad argument"):
        nw.rollout_policy_mlp(w_ptrs, 64, 4, categorical=True, mappo=(4, 1e-5))
    with pytest.raises(MpeError, match="bad argument"):
        nw.rollout_policy_mlp(w_ptrs, 64, 4, categorical=True, mappo=(0, float("nan")))
    unchanged(env, before, epoch)
    wc = make_product_env("simple_world_comm", num_envs=64, seed=9)   # a program without the kernel
    wc.reset()
    wnw = wc.world.native
    wbefore, wepoch = state(wc), wnw.epoch
    for kw in ({}, {"episode_length": 2}):
        with pytest.raises(MpeError, match="no compiled"):
            wc.rollout_policy(make_mappo_actors(wnw.obs_dims, wnw.act_dims, True, False), 4, explore_seed=1,
                              action_mode="categorical", record_log_probs=True, **kw)
        unchanged(wc, wbefore, wepoch)
