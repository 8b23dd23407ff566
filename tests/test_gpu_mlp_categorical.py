"""env.rollout_policy(..., action_mode="categorical") with MADDPG's two-hidden-layer actor
(mpe_rollout_policy_mlp_categorical and its episode form): every agent applies the one-hot vector of the arg-max of its
(Gumbel-perturbed) logits per action sub-space and records the index and the log-probability, the experience a
policy-gradient trainer (PPO, A2C) stores.  Checked for every program the kernel is built for, at both hidden widths,
exploring and greedy: replay of the recorded indices as one-hot vectors through fused steps of a twin env, bit for bit;
every pick and log-probability against the float64 model of the TF32 actor; the sample distribution; agreement with the
default mode's Gumbel-softmax sample; the index convention; the episode form against its loop; the interface."""
import numpy as np
import pytest

from helpers import device_sms, launch_shape, make_product_env, regime_size
from mlp_categorical_helpers import (bounds, categorical_pick, explain_categorical_mismatches, log_softmax_at,
                                     one_hot_torch)
from mlp_helpers import actor_logits, gumbel_noise, segment_softmax
from mlp_programs import PROGRAMS, as_sequential, make_policies, mlp_block_cap, state, twins

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

# Against the unrounded float64 actor a log-probability is not held to the probabilities' 5e-3 (LOOSE_MAX of
# tests/test_gpu_mlp_policy.py): it moves with the logits, by up to 2 max |dz| per sub-space, and measures up to 8e-3 at
# H = 32.  The bound is computed per row from the TF32 model's logit error instead.
LOGP_FLIP_SLACK = 1e-3
RECORDS = dict(record_actions=True, per_step_rewards=True, record_observations=True, record_log_probs=True)


def segments_of(env):
    d = env.world.native.desc
    return [([5] if d.agent_movable[i] else []) + ([d.dim_c] if not d.agent_silent[i] else []) for i in range(env.n)]


def stride_of(act_dims):
    return 2 if max(act_dims) <= 8 else 4


def size(tag, H, wpb, base=None, episodes=False):
    cap = mlp_block_cap(tag, H, episodes, categorical=True)
    sms = device_sms()
    n = regime_size("mlp", sms, min(wpb, cap), cap=cap, base=base)
    assert launch_shape("mlp", n, sms, cap)[0] == min(wpb, cap)
    return n


def observe(env):
    nw = env.world.native
    return [o.clone() for o in nw.observe(out=nw.new_outputs(), flags=env._flags()).obs]


def check_replay_and_numerics(tag, H, n, T, explore, check_numerics=True):
    """(1) the index records, as one-hot vectors, fed to T fused steps of a twin env reproduce state, comm state, final
    observations, every step's rewards and their sums bit for bit, the observation records are the twin's observations,
    and immovable agents never move; (2) every pick is the arg-max of the float64 TF32 model (+ the float64 Gumbel
    noise) and every log-probability its log_softmax at the pick to 1e-5, unless a TF32 rounding flip or the Gumbel
    gap explains the row; against the unrounded float64 actor every log-probability is within twice the TF32 model's
    largest logit error per sub-space (plus LOGP_FLIP_SLACK)"""
    env_a, env_b = twins(tag, n)
    na, nb = env_a.world.native, env_b.world.native
    A, act_dims, segs = env_a.n, list(na.act_dims), segments_of(env_a)
    pv0 = na.agent_pv.clone()
    pols = make_policies(na.obs_dims, act_dims, H)
    seed = 0x1234_5678_9ABC if explore else None
    obs_b = observe(env_b)
    obs_r, rew_r, done_r, _, ex = env_a.rollout_policy(pols, T, explore_seed=seed, action_mode="categorical", **RECORDS)
    idx, logp, rew_steps, obs_rec = ex["actions"], ex["log_probs"], ex["rewards"], ex["observations"]
    assert [(tuple(k.shape), k.dtype) for k in idx] == [((T, n, len(s)), torch.int32) for s in segs]
    assert tuple(logp.shape) == (T, A, n) and logp.dtype == torch.float32
    assert env_a.explore_epoch == (1 if explore else 0)
    pols_np = [[t.cpu().numpy() for t in p] for p in pols]
    rew_sum = torch.zeros(A, n, device="cuda")
    flips = gaps = 0
    lmax = 0.0
    for t in range(T):
        for i in range(A):
            assert torch.equal(obs_rec[i][t], obs_b[i]), (t, i)
            if not check_numerics:
                continue
            o = obs_b[i].cpu().numpy()
            g = gumbel_noise(seed, 0, np.arange(n), t, i, A, n_logits=act_dims[i], stride=stride_of(act_dims)) \
                if explore else 0.0
            k = idx[i][t].cpu().numpy()
            lp = logp[t, i].cpu().numpy().astype(np.float64)
            f, gp = explain_categorical_mismatches(k, lp, o, pols_np[i], segs[i], noise=g)
            flips, gaps = flips + f, gaps + gp
            z64 = actor_logits(o, *pols_np[i], tf32=False)
            err = np.abs(lp - log_softmax_at(z64, k, segs[i]))
            lmax = max(lmax, float(err.max()))
            # log_softmax(z)[k] moves by at most 2 max_c |dz_c| per sub-space: the TF32 error of the logits, plus what
            # a rounding flip adds (a few 1e-4)
            dz = np.abs(actor_logits(o, *pols_np[i], tf32=True) - z64)
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
    if check_numerics:
        print("\ncategorical %s H=%d n=%d explore=%s: %d of %d rows explained by TF32 rounding flips, %d by the Gumbel "
              "gap; log-probabilities within %.3e of the unrounded actor" % (tag, H, n, explore, flips, n * T * A, gaps,
                                                                              lmax))


@pytest.mark.parametrize("tag", tuple(PROGRAMS))
@pytest.mark.parametrize("H", [32, 64])
@pytest.mark.parametrize("explore", [True, False])
def test_categorical_replay_and_numerics(tag, H, explore):
    """a ragged multi-warp launch: min(5, cap)-warp blocks with a partial last block and a partial last warp"""
    check_replay_and_numerics(tag, H, size(tag, H, 5), 3, explore)


@pytest.mark.parametrize("tag,H,explore", [("simple_spread_n3", 64, True), ("simple_speaker_listener", 32, True),
                                           ("simple_reference", 64, False), ("simple_tag_6v2", 64, True),
                                           ("simple_spread_n6", 32, False)])
def test_categorical_replay_at_the_block_cap(tag, H, explore):
    """65 536 worlds plus a ragged tail in blocks at the categorical kernel's cap"""
    check_replay_and_numerics(tag, H, size(tag, H, 16, base=65536), 2, explore)


def _fixed_logit_policies(env, H, b3_of):
    nw = env.world.native
    out = []
    for i, (W1, b1, W2, b2, W3, b3) in enumerate(make_policies(nw.obs_dims, nw.act_dims, H)):
        fixed = b3_of(i)
        if fixed is not None:
            W3, b3 = torch.zeros_like(W3), torch.tensor(fixed, dtype=torch.float32, device="cuda")
        out.append((W1, b1, W2, b2, W3, b3))
    return out


def test_speaker_utterances_follow_softmax_of_fixed_logits():
    """W3 = 0: the speaker's categorical utterance is a draw from softmax(b3); chi-square over 65 536 worlds x 2 steps
    with fixed seeds"""
    from scipy.stats import chisquare
    n, T = 65536, 2
    env = make_product_env("simple_speaker_listener", num_envs=n, seed=4)
    env.reset()
    b3 = [0.4, -0.6, 0.9]
    pols = _fixed_logit_policies(env, 32, lambda i: b3 if i == 0 else None)
    ex = env.rollout_policy(pols, T, record_actions=True, explore_seed=2024, action_mode="categorical")[4]
    k = ex["actions"][0][..., 0].reshape(-1).cpu().numpy()
    counts = np.bincount(k, minlength=3)
    expect = segment_softmax(np.asarray(b3, np.float64)) * k.size
    _, p = chisquare(counts, expect)
    print("\nspeaker utterances %s, expected %s, p = %.3g" % (counts, expect.round(1), p))
    assert p > 1e-3, (counts, expect, p)


def test_reference_subspaces_are_independent_draws():
    """simple_reference (movement and utterance logits of one agent, W3 = 0): the (movement, utterance) table of agent 0
    follows the product of the two softmaxes; chi-square over 65 536 worlds x 2 steps"""
    from scipy.stats import chisquare
    n, T = 65536, 2
    env = make_product_env("simple_reference", num_envs=n, seed=4)
    env.reset()
    move = [0.3, -0.2, 0.5, -0.7, 0.1]
    utter = [0.2, -0.4, 0.6, 0.0, -0.3, 0.45, -0.1, 0.35, -0.5, 0.05]
    pols = _fixed_logit_policies(env, 32, lambda i: move + utter)
    ex = env.rollout_policy(pols, T, record_actions=True, explore_seed=77, action_mode="categorical")[4]
    k = ex["actions"][0].reshape(-1, 2).cpu().numpy()
    counts = np.bincount(k[:, 0] * 10 + k[:, 1], minlength=50)
    expect = np.outer(segment_softmax(np.asarray(move)), segment_softmax(np.asarray(utter))).reshape(-1) * k.shape[0]
    _, p = chisquare(counts, expect)
    print("\nreference (movement, utterance) table: p = %.3g" % p)
    assert p > 1e-3, p


@pytest.mark.parametrize("tag", ["simple_spread_n3", "simple_speaker_listener", "simple_reference", "simple_crypto",
                                 "simple_tag_6v2", "simple_push"])
@pytest.mark.parametrize("H", [32, 64])
def test_categorical_pick_is_the_argmax_of_the_default_sample(tag, H):
    """T = 1 from the same state with the same seed and epoch: the categorical index of every sub-space is the arg-max
    of the default mode's Gumbel-softmax action, except where two of that row's probabilities are equal in fp32"""
    n = size(tag, H, 5)
    env_a, env_b = twins(tag, n)
    segs = segments_of(env_a)
    pols = make_policies(env_a.world.native.obs_dims, env_a.world.native.act_dims, H)
    ka = env_a.rollout_policy(pols, 1, record_actions=True, explore_seed=31, action_mode="categorical")[4]["actions"]
    pb = env_b.rollout_policy(pols, 1, record_actions=True, explore_seed=31)[4]["actions"]
    torch.cuda.synchronize()
    ties = 0
    for i, s in enumerate(segs):
        k = ka[i][0].cpu().numpy()
        pr = pb[i][0].cpu().numpy()
        want = categorical_pick(pr, s)
        for r, c in zip(*np.where(k != want)):
            a = sum(s[:c])
            assert pr[r, a + k[r, c]] == pr[r, a + want[r, c]], (i, r, c)     # an fp32 tie of the probabilities
            ties += 1
    print("\n%s H=%d: %d sub-space picks differ from the arg-max of the Gumbel-softmax sample, all fp32 ties"
          % (tag, H, ties))


def test_index_one_moves_plus_x_and_is_not_the_discrete_input_code():
    """index 1 of the movement segment is +x (the one-hot convention); the same indices fed through
    env.discrete_action_input (where 1 is -x) do not reproduce the state"""
    n = 1031
    env_a, env_b = twins("simple", n)
    nw = env_a.world.native
    pols = _fixed_logit_policies(env_a, 32, lambda i: [0.0, 4.0, 0.0, 0.0, 0.0])
    ex = env_a.rollout_policy(pols, 1, record_actions=True, action_mode="categorical")[4]
    k = ex["actions"][0]
    assert bool((k == 1).all())
    v = nw.agent_pv[0, :, 2:4]
    assert bool((v[:, 0] > 0).all()) and bool((v[:, 1] == 0).all())
    env_b.discrete_action_input = True
    env_b.step([k[0]])
    torch.cuda.synchronize()
    assert bool((env_b.world.native.agent_pv[0, :, 2] < 0).all())
    assert not torch.equal(nw.agent_pv, env_b.world.native.agent_pv)


def categorical_loop(env, pols, E, L, seed):
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
@pytest.mark.parametrize("H", [32, 64])
@pytest.mark.parametrize("E,L,explore", [(3, 4, True), (2, 3, False)])
def test_categorical_episodes_equal_the_loop(tag, H, E, L, explore):
    n = size(tag, H, 5, episodes=True)
    env_a, env_b = twins(tag, n)
    nw = env_a.world.native
    pols = make_policies(nw.obs_dims, nw.act_dims, H)
    seed = 21 if explore else None
    epoch = nw.epoch
    obs, ret, done, _, ex = env_a.rollout_policy(pols, E * L, episode_length=L, explore_seed=seed,
                                                 action_mode="categorical", **RECORDS)
    ref = categorical_loop(env_b, pols, E, L, seed)
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


@pytest.mark.parametrize("tag", ["simple_spread_n3", "simple_reference"])
def test_sequential_actors_equal_tuples_and_a_seed_reproduces(tag):
    env_a, env_b = twins(tag, 1031)
    nw = env_a.world.native
    pols = make_policies(nw.obs_dims, nw.act_dims, 64)
    ra = env_a.rollout_policy(pols, 5, explore_seed=2, action_mode="categorical", **RECORDS)
    rb = env_b.rollout_policy(as_sequential(pols), 5, explore_seed=2, action_mode="categorical", **RECORDS)
    torch.cuda.synchronize()
    for x, y in zip(ra[0] + ra[1], rb[0] + rb[1]):
        assert torch.equal(x, y)
    for key in ("rewards", "log_probs"):
        assert torch.equal(ra[4][key], rb[4][key]), key
    for key in ("actions", "observations"):
        for x, y in zip(ra[4][key], rb[4][key]):
            assert torch.equal(x, y), key
    assert env_a.explore_epoch == 1
    # the same seed and epoch from the same state reproduce every record; the next epoch draws other samples
    env_c = make_product_env(tag, num_envs=1031, seed=9)
    env_c.reset()
    rc = env_c.rollout_policy(pols, 5, explore_seed=2, action_mode="categorical", **RECORDS)
    rd = env_c.rollout_policy(pols, 5, explore_seed=2, action_mode="categorical", **RECORDS)
    assert env_c.explore_epoch == 2
    torch.cuda.synchronize()
    assert torch.equal(rc[4]["log_probs"], ra[4]["log_probs"])
    for x, y in zip(rc[4]["actions"], ra[4]["actions"]):
        assert torch.equal(x, y)
    assert not all(torch.equal(x, y) for x, y in zip(rd[4]["actions"], rc[4]["actions"]))
    # greedy calls leave the exploration epoch where it is
    env_c.rollout_policy(pols, 2, action_mode="categorical")
    assert env_c.explore_epoch == 2


@pytest.mark.parametrize("tag", ["simple_spread_n3", "simple_speaker_listener"])
def test_sharded_categorical_equals_the_full_batch(tag):
    n, T = 1031, 4
    full = make_product_env(tag, num_envs=n, seed=9)
    full.reset()
    nw = full.world.native
    pols = make_policies(nw.obs_dims, nw.act_dims, 32)
    ex = full.rollout_policy(pols, T, explore_seed=77, action_mode="categorical", **RECORDS)[4]
    lo = 0
    for rank in range(2):
        sh = make_product_env(tag, num_envs=n, seed=9, rank=rank, world_size=2)
        sh.reset()
        m = sh.world.native.n_env
        ex_s = sh.rollout_policy(pols, T, explore_seed=77, action_mode="categorical", **RECORDS)[4]
        torch.cuda.synchronize()
        for x, y in zip(ex_s["actions"], ex["actions"]):
            assert torch.equal(x, y[:, lo:lo + m])
        assert torch.equal(ex_s["log_probs"], ex["log_probs"][:, :, lo:lo + m])
        lo += m
    assert lo == n


def test_records_are_none_unless_requested():
    env = make_product_env("simple_speaker_listener", num_envs=100, seed=9)
    env.reset()
    nw = env.world.native
    pols = make_policies(nw.obs_dims, nw.act_dims, 32)
    ex = env.rollout_policy(pols, 3, action_mode="categorical")[4]
    assert ex == {"actions": None, "rewards": None, "observations": None, "log_probs": None}
    ex = env.rollout_policy(pols, 4, episode_length=2, action_mode="categorical")[4]
    assert ex == {"actions": None, "rewards": None, "observations": None, "log_probs": None,
                  "final_observations": None}
    ex = env.rollout_policy(pols, 3, record_log_probs=True, action_mode="categorical")[4]
    assert ex["actions"] is None and tuple(ex["log_probs"].shape) == (3, env.n, 100)
    ex = env.rollout_policy(pols, 3, record_actions=True)[4]      # the default mode keeps its keys
    assert set(ex) == {"actions", "rewards", "observations"} and ex["actions"][0].dtype == torch.float32


def test_refusals_leave_state_and_epochs_unchanged():
    from multiagent_particle_envs_b200._lib import MpeError
    env = make_product_env("simple_spread_n3", num_envs=64, seed=9)
    env.reset()
    nw = env.world.native
    before, epoch = state(env), nw.epoch
    pols = make_policies(nw.obs_dims, nw.act_dims, 32)

    def unchanged(e, b, ep):
        torch.cuda.synchronize()
        for x, y in zip(state(e), b):
            assert torch.equal(x, y)
        assert e.world.native.epoch == ep and e.explore_epoch == 0

    with pytest.raises(ValueError, match="action_mode"):
        env.rollout_policy(pols, 4, explore_seed=1, action_mode="argmax")
    unchanged(env, before, epoch)
    with pytest.raises(ValueError, match="record_log_probs"):
        env.rollout_policy(pols, 4, explore_seed=1, record_log_probs=True)
    unchanged(env, before, epoch)
    one_layer = [torch.nn.Sequential(torch.nn.Linear(od, 32), torch.nn.ReLU(), torch.nn.Linear(32, 5)).cuda()
                 for od in nw.obs_dims]
    with pytest.raises(NotImplementedError, match="categorical"):
        env.rollout_policy(one_layer, 4, action_mode="categorical")
    unchanged(env, before, epoch)
    with pytest.raises(ValueError, match="episode_length"):
        env.rollout_policy(pols, 7, episode_length=2, action_mode="categorical")
    unchanged(env, before, epoch)
    # (t * 8 + i) * 2 + b must stay below the tag bit 2^30: tag 6+2 at 2^26 + 1 steps, in both forms
    tag = make_product_env("simple_tag_6v2", num_envs=64, seed=9)
    tag.reset()
    tnw = tag.world.native
    tbefore, tepoch = state(tag), tnw.epoch
    tpols = make_policies(tnw.obs_dims, tnw.act_dims, 32)
    for kw in ({}, {"episode_length": 2 ** 26 + 1}):
        with pytest.raises(MpeError, match="bad argument"):
            tag.rollout_policy(tpols, 2 ** 26 + 1, explore_seed=1, action_mode="categorical", **kw)
        unchanged(tag, tbefore, tepoch)
    wc = make_product_env("simple_world_comm", num_envs=64, seed=9)   # a program without the kernel
    wc.reset()
    wnw = wc.world.native
    wbefore, wepoch = state(wc), wnw.epoch
    for kw in ({}, {"episode_length": 2}):
        with pytest.raises(MpeError, match="no compiled"):
            wc.rollout_policy(make_policies(wnw.obs_dims, wnw.act_dims, 32), 4, explore_seed=1,
                              action_mode="categorical", record_log_probs=True, **kw)
        unchanged(wc, wbefore, wepoch)
