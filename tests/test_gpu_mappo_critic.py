"""env.rollout_policy(mappo_actors, T, action_mode="categorical", critic=...) (mpe_rollout_policy_mappo_critic and its
episode form): MAPPO's centralized critic on share_obs inside the rollout kernel.  For every program with a critic
kernel, shared and (where they fit) per-agent critics, ReLU and tanh, exploring and greedy, the input LayerNorm on for
half of the cases: every output, record, the state and both epochs bit-identical to the same call without a critic;
every value teacher-forced on the observation records against the float64 model of the kernel's recipe (the flip-free
bound, or a TF32 rounding flip) and against the unfolded float64 critic (LOOSE); the final values on the returned or
final observations; a shared critic against per-agent copies; the episode form against its loop; the refusals."""
import copy

import numpy as np
import pytest

from critic_helpers import (CRITIC_PROGRAMS, LOOSE, CriticModel, critic_block_cap, critic_smem_warps,
                            explain_value_mismatches, make_critic, module_values, share_obs)
from helpers import device_sms, launch_shape, make_product_env, regime_size
from mappo_helpers import FEATURE_NORM, TANH, make_mappo_actors
from mlp_programs import state, twins

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

RECORDS = dict(record_actions=True, per_step_rewards=True, record_observations=True, record_log_probs=True)
# per-agent critics fit next to the actors for these programs (critic_smem_warps(tag, n) >= 1)
PER_AGENT = ("simple", "simple_spread_n2", "simple_spread_n3", "simple_tag_1v1", "simple_tag_2v1", "simple_adversary",
             "simple_push", "simple_speaker_listener", "simple_reference", "simple_crypto")
CASES = [(t, m) for t in CRITIC_PROGRAMS for m in (("shared", "per_agent") if t in PER_AGENT and t != "simple"
                                                  else ("shared",))]


def size(tag, wpb, base=None, episodes=False, count=1):
    cap = min(critic_block_cap(tag, episodes), critic_smem_warps(tag, count))
    sms = device_sms()
    n = regime_size("mlp", sms, min(wpb, cap), cap=cap, base=base)
    assert launch_shape("mlp", n, sms, cap)[0] == min(wpb, cap)
    return n


def critics_for(nw, mode, tanh, fn):
    if mode == "shared":
        return make_critic(nw.obs_dims, tanh, fn)
    return [make_critic(nw.obs_dims, tanh, fn, seed=11 + i) for i in range(len(nw.obs_dims))]


def models_of(critic, nw):
    from multiagent_particle_envs_b200.environment import mappo_critic_params
    params, tanh, fn, eps = mappo_critic_params(critic, nw.obs_dims)
    net = ((FEATURE_NORM if fn else 0) | (TANH if tanh else 0), eps)
    return [CriticModel([t.to(torch.float32).cpu().numpy() for t in p], net, nw.obs_dims) for p in params]


def compare_outputs(ra, rb, env_a, env_b, keys=("actions", "observations")):
    """(obs, rew, done, info, extras) of two calls and the two envs' state: bit-identical"""
    torch.cuda.synchronize()
    for x, y in zip(ra[0] + ra[1] + ra[2], rb[0] + rb[1] + rb[2]):
        assert torch.equal(x, y)
    for key in ("rewards", "log_probs"):
        assert torch.equal(ra[4][key], rb[4][key]), key
    for key in keys:
        for x, y in zip(ra[4][key], rb[4][key]):
            assert torch.equal(x, y), key
    for x, y in zip(state(env_a), state(env_b)):
        assert torch.equal(x, y)
    assert env_a.world.native.epoch == env_b.world.native.epoch and env_a.explore_epoch == env_b.explore_epoch


def check_values(values, obs_lists, models, critics, A, rows=None):
    """values [S, A, n] against the models on share_obs rows of obs_lists (S lists of A [n, obs_dim_i] tensors); rows
    (an index array, or None for all) selects the worlds checked"""
    flips, loose = 0, 0.0
    mods = critics if isinstance(critics, list) else [critics]
    sel = slice(None) if rows is None else rows
    for s, obs in enumerate(obs_lists):
        x = share_obs([o.cpu().numpy()[sel] for o in obs])
        for i in range(A):
            k = i if len(models) > 1 else 0
            got = values[s, i].cpu().numpy()[sel].astype(np.float64)
            if len(models) == 1 and i > 0:
                assert torch.equal(values[s, i], values[s, 0])          # the shared value, written for every agent
                continue
            flips += explain_value_mismatches(got, x, models[k])
            err = np.abs(got - module_values(mods[k], x))
            loose = max(loose, float(err.max()))
            assert (err <= LOOSE).all(), (s, i, float(err.max()))
    return flips, loose


@pytest.mark.parametrize("tag,mode", CASES)
@pytest.mark.parametrize("tanh", [False, True])
@pytest.mark.parametrize("explore", [True, False])
def test_critic_changes_nothing_and_values_match_the_model(tag, mode, tanh, explore):
    """a ragged multi-warp launch (2-warp blocks, a partial last block and warp); the input LayerNorm is on for (ReLU,
    exploring) and (tanh, greedy)"""
    fn = explore != tanh
    count = 1 if mode == "shared" else len(make_product_env(tag, num_envs=1).world.native_shapes().obs_dims)
    n, T = size(tag, 2, count=count), 3
    env_a, env_b = twins(tag, n)
    nw = env_a.world.native
    A = env_a.n
    pols = make_mappo_actors(nw.obs_dims, nw.act_dims, tanh, fn)
    critic = critics_for(nw, mode, tanh, fn)
    seed = 0x5EED if explore else None
    ra = env_a.rollout_policy(pols, T, explore_seed=seed, action_mode="categorical", critic=critic, **RECORDS)
    rb = env_b.rollout_policy(pols, T, explore_seed=seed, action_mode="categorical", **RECORDS)
    compare_outputs(ra, rb, env_a, env_b)
    assert "values" not in rb[4]
    values, final = ra[4]["values"], ra[4]["final_values"]
    assert tuple(values.shape) == (T, A, n) and values.dtype == torch.float32
    assert tuple(final.shape) == (A, n) and final.dtype == torch.float32
    models = models_of(critic, nw)
    obs_rec = ra[4]["observations"]
    flips, loose = check_values(values, [[obs_rec[i][t] for i in range(A)] for t in range(T)], models, critic, A)
    f2, l2 = check_values(final[None], [list(ra[0])], models, critic, A)
    print("\ncritic %s %s tanh=%s feature_norm=%s n=%d: %d of %d values explained by TF32 rounding flips; within %.2e "
          "of the unfolded float64 critic" % (tag, mode, tanh, fn, n, flips + f2, n * (T + 1) * len(models),
                                               max(loose, l2)))


@pytest.mark.parametrize("tag,mode,tanh", [("simple_spread_n3", "shared", False),
                                           ("simple_speaker_listener", "per_agent", True)])
def test_critic_at_the_block_cap(tag, mode, tanh):
    """65 536 worlds plus a ragged tail in blocks at the cap the critics' count leaves: every output bit-identical, the
    values of every 16th world and of the last block's worlds against the model"""
    count = 1 if mode == "shared" else 2
    n = size(tag, 64, base=65536, count=count)
    env_a, env_b = twins(tag, n)
    nw = env_a.world.native
    pols = make_mappo_actors(nw.obs_dims, nw.act_dims, tanh, True)
    critic = critics_for(nw, mode, tanh, True)
    ra = env_a.rollout_policy(pols, 2, explore_seed=3, action_mode="categorical", critic=critic, **RECORDS)
    rb = env_b.rollout_policy(pols, 2, explore_seed=3, action_mode="categorical", **RECORDS)
    compare_outputs(ra, rb, env_a, env_b)
    obs_rec = ra[4]["observations"]
    rows = np.unique(np.concatenate([np.arange(0, n, 16), np.arange(n - 32 * 12, n)]))
    check_values(ra[4]["values"], [[o[t] for o in obs_rec] for t in range(2)], models_of(critic, nw), critic, env_a.n,
                 rows=rows)
    check_values(ra[4]["final_values"][None], [list(ra[0])], models_of(critic, nw), critic, env_a.n, rows=rows)


@pytest.mark.parametrize("tag,mode", [("simple_spread_n3", "shared"), ("simple_spread_n3", "per_agent"),
                                      ("simple_tag", "shared"), ("simple_speaker_listener", "per_agent"),
                                      ("simple_reference", "shared"), ("simple_spread_n5", "shared")])
@pytest.mark.parametrize("E,L,explore,tanh,fn", [(3, 4, True, True, True), (2, 3, False, False, False)])
def test_episode_form(tag, mode, E, L, explore, tanh, fn):
    """the episode form with a critic: everything else as without it; values and final values against the model; and
    bit for bit its loop of single-episode calls each followed by reset()"""
    count = 1 if mode == "shared" else len(make_product_env(tag, num_envs=1).world.native_shapes().obs_dims)
    n = size(tag, 2, episodes=True, count=count)
    env_a, env_b = twins(tag, n)
    env_c = twins(tag, n)[0]
    nw = env_a.world.native
    A = env_a.n
    pols = make_mappo_actors(nw.obs_dims, nw.act_dims, tanh, fn)
    critic = critics_for(nw, mode, tanh, fn)
    seed = 21 if explore else None
    kw = dict(episode_length=L, explore_seed=seed, action_mode="categorical", **RECORDS)
    ra = env_a.rollout_policy(pols, E * L, critic=critic, **kw)
    rb = env_b.rollout_policy(pols, E * L, **kw)
    compare_outputs(ra, rb, env_a, env_b, keys=("actions", "observations", "final_observations"))
    values, final = ra[4]["values"], ra[4]["final_values"]
    assert tuple(values.shape) == (E * L, A, n) and tuple(final.shape) == (E, A, n)
    models = models_of(critic, nw)
    obs_rec, fin = ra[4]["observations"], ra[4]["final_observations"]
    check_values(values, [[o[t] for o in obs_rec] for t in range(E * L)], models, critic, A)
    check_values(final, [[f[e] for f in fin] for e in range(E)], models, critic, A)
    # the loop
    lv, lf = [], []
    for _ in range(E):
        _, _, _, _, ex = env_c.rollout_policy(pols, L, explore_seed=seed, action_mode="categorical", critic=critic,
                                              **RECORDS)
        lv.append(ex["values"])
        lf.append(ex["final_values"])
        env_c.reset()
    torch.cuda.synchronize()
    assert torch.equal(values, torch.cat(lv)) and torch.equal(final, torch.stack(lf))
    for x, y in zip(state(env_a), state(env_c)):
        assert torch.equal(x, y)


@pytest.mark.parametrize("tag", ["simple_spread_n3", "simple_speaker_listener", "simple_crypto"])
def test_a_shared_critic_equals_per_agent_copies(tag):
    env_a, env_b = twins(tag, 1031)
    nw = env_a.world.native
    pols = make_mappo_actors(nw.obs_dims, nw.act_dims, True, True)
    critic = make_critic(nw.obs_dims, True, True)
    ra = env_a.rollout_policy(pols, 5, explore_seed=2, action_mode="categorical", critic=[critic] * env_a.n, **RECORDS)
    rb = env_b.rollout_policy(pols, 5, explore_seed=2, action_mode="categorical",
                              critic=[copy.deepcopy(critic) for _ in range(env_a.n)], **RECORDS)
    compare_outputs(ra, rb, env_a, env_b)
    assert torch.equal(ra[4]["values"], rb[4]["values"]) and torch.equal(ra[4]["final_values"], rb[4]["final_values"])


def test_refusals_leave_state_and_epochs_unchanged():
    from multiagent_particle_envs_b200._lib import MpeError

    def env_of(tag):
        env = make_product_env(tag, num_envs=64, seed=9)
        env.reset()
        return env, state(env), env.world.native.epoch

    def unchanged(e, b, ep):
        torch.cuda.synchronize()
        for x, y in zip(state(e), b):
            assert torch.equal(x, y)
        assert e.world.native.epoch == ep and e.explore_epoch == 0

    # no critic kernel, or per-agent critics that do not fit in shared memory
    for tag, per_agent in (("simple_spread_n6", False), ("simple_tag_6v2", False), ("simple_spread_n4", True),
                           ("simple_spread_n5", True), ("simple_tag", True), ("simple_tag_4v2", True),
                           ("simple_adversary_n4", True)):
        env, before, epoch = env_of(tag)
        nw = env.world.native
        pols = make_mappo_actors(nw.obs_dims, nw.act_dims, False, True)
        critic = critics_for(nw, "per_agent" if per_agent else "shared", False, True)
        for kw in ({}, {"episode_length": 2}):
            with pytest.raises(MpeError, match="no compiled"):
                env.rollout_policy(pols, 4, explore_seed=1, action_mode="categorical", critic=critic, **kw)
            unchanged(env, before, epoch)
    # a critic that is not the actors' kind, or malformed
    env, before, epoch = env_of("simple_spread_n3")
    nw = env.world.native
    pols = make_mappo_actors(nw.obs_dims, nw.act_dims, False, True)
    for critic, match in ((make_critic(nw.obs_dims, True, True), "activation"),
                          (make_critic(nw.obs_dims, False, False), "input LayerNorm"),
                          (make_critic(nw.obs_dims, False, True, eps=1e-3), "eps"),
                          (make_critic(nw.obs_dims[:2], False, True), "expected Linear weights"),
                          ([make_critic(nw.obs_dims, False, True)] * 2, "list of 1 or 3")):
        with pytest.raises(ValueError, match=match):
            env.rollout_policy(pols, 4, explore_seed=1, action_mode="categorical", critic=critic)
        unchanged(env, before, epoch)
    with pytest.raises(NotImplementedError, match="critic"):
        env.rollout_policy(pols, 4, critic=make_critic(nw.obs_dims, False, True))
    unchanged(env, before, epoch)
