"""env.rollout_policy(..., critic=..., centralized_critic=False): IPPO's local critics.

MLP (mpe_rollout_policy_mappo_local_critic[_episodes]), shared and per-agent, ReLU and tanh, the input LayerNorm on and
off, exploring and greedy, at production launch shapes and at the block cap: every other output, the state and both
epochs bit-identical to the same call without a critic; every value V_k(obs_k) against the float64 model of the
kernel's recipe on [obs_k] (the flip-free bound, or a TF32 rounding flip) and within LOOSE of the unfolded module; on
simple the local and centralized critics bit-identical; spread N=6 with its shared critic; the episode form against its
loop.  Recurrent (mpe_critic_gru_local): values per agent within LOOSE of the modules run free from h0[k]; hidden
states carried over; episodes against the loop; determinism; on simple bit-identical to mpe_critic_gru.  GAE with a
per-agent ValueNorm over IPPO's values; the MpeError refusals leave state and epochs unchanged."""
import numpy as np
import pytest

from critic_helpers import LOOSE, explain_value_mismatches, make_critic, module_values
from gae_helpers import gae_mirror
from helpers import device_sms, launch_shape, make_product_env, regime_size
from ippo_helpers import (LOCAL_PROGRAMS, local_critic_block_cap, local_critic_smem_warps, local_models,
                          make_local_critics, make_rcritic, shared_ok)
from mappo_helpers import make_mappo_actors
from mlp_programs import shapes_of, state, twins
from rcritic_helpers import H, module_rollout
from rmappo_helpers import make_rmappo_actor
from test_gpu_mappo_critic import compare_outputs

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

RECORDS = dict(record_actions=True, per_step_rewards=True, record_observations=True, record_log_probs=True)
LOCAL = dict(action_mode="categorical", centralized_critic=False)
CASES = [(t, m) for t in LOCAL_PROGRAMS for m in ("shared", "per_agent")
         if (m == "shared" and shared_ok(t)) or (m == "per_agent" and t != "simple"
                                                 and local_critic_smem_warps(t, len(shapes_of(t)[0])) >= 1)]


def count_of(tag, mode):
    return 1 if mode == "shared" else len(shapes_of(tag)[0])


def size(tag, wpb, base=None, episodes=False, count=1):
    cap = min(local_critic_block_cap(tag, episodes), local_critic_smem_warps(tag, count))
    sms = device_sms()
    n = regime_size("mlp", sms, min(wpb, cap), cap=cap, base=base)
    assert launch_shape("mlp", n, sms, cap)[0] == min(wpb, cap)
    return n


def check_values(values, obs_lists, critic, obs_dims, rows=None):
    """values [S, A, n] against agent k's model and module on obs_k of obs_lists (S lists of A [n, obs_dim_k])"""
    models, mods = local_models(critic, obs_dims)
    flips, loose = 0, 0.0
    sel = slice(None) if rows is None else rows
    for s, obs in enumerate(obs_lists):
        for k in range(len(obs_dims)):
            x = obs[k].cpu().numpy()[sel].astype(np.float64)
            got = values[s, k].cpu().numpy()[sel].astype(np.float64)
            flips += explain_value_mismatches(got, x, models[k])
            err = np.abs(got - module_values(mods[k], x))
            loose = max(loose, float(err.max()))
            assert (err <= LOOSE).all(), (s, k, float(err.max()))
    return flips, loose


@pytest.mark.parametrize("tag,mode", CASES)
@pytest.mark.parametrize("tanh", [False, True])
@pytest.mark.parametrize("explore", [True, False])
def test_local_critic_changes_nothing_and_values_match_the_model(tag, mode, tanh, explore):
    """a ragged multi-warp launch (2-warp blocks); the input LayerNorm is on for (ReLU, exploring) and (tanh, greedy)"""
    fn = explore != tanh
    n, T = size(tag, 2, count=count_of(tag, mode)), 3
    env_a, env_b = twins(tag, n)
    nw = env_a.world.native
    A = env_a.n
    pols = make_mappo_actors(nw.obs_dims, nw.act_dims, tanh, fn)
    critic = make_local_critics(nw.obs_dims, mode, tanh, fn)
    seed = 0x5EED if explore else None
    ra = env_a.rollout_policy(pols, T, explore_seed=seed, critic=critic, **LOCAL, **RECORDS)
    rb = env_b.rollout_policy(pols, T, explore_seed=seed, action_mode="categorical", **RECORDS)
    compare_outputs(ra, rb, env_a, env_b)
    values, final = ra[4]["values"], ra[4]["final_values"]
    assert tuple(values.shape) == (T, A, n) and tuple(final.shape) == (A, n)
    obs_rec = ra[4]["observations"]
    flips, loose = check_values(values, [[obs_rec[k][t] for k in range(A)] for t in range(T)], critic, nw.obs_dims)
    f2, l2 = check_values(final[None], [list(ra[0])], critic, nw.obs_dims)
    print("\nlocal critic %s %s tanh=%s feature_norm=%s n=%d: %d values explained by TF32 rounding flips; within %.2e "
          "of the unfolded float64 critic" % (tag, mode, tanh, fn, n, flips + f2, max(loose, l2)))


@pytest.mark.parametrize("tag,mode,tanh", [("simple_spread_n3", "per_agent", False), ("simple_spread_n6", "shared", True),
                                           ("simple_speaker_listener", "per_agent", True)])
def test_local_critic_at_the_block_cap(tag, mode, tanh):
    """65 536 worlds plus a ragged tail in blocks at the cap: every output bit-identical, the values of every 16th
    world and of the last block's worlds against the model"""
    n = size(tag, 64, base=65536, count=count_of(tag, mode))
    env_a, env_b = twins(tag, n)
    nw = env_a.world.native
    pols = make_mappo_actors(nw.obs_dims, nw.act_dims, tanh, True)
    critic = make_local_critics(nw.obs_dims, mode, tanh, True)
    ra = env_a.rollout_policy(pols, 2, explore_seed=3, critic=critic, **LOCAL, **RECORDS)
    rb = env_b.rollout_policy(pols, 2, explore_seed=3, action_mode="categorical", **RECORDS)
    compare_outputs(ra, rb, env_a, env_b)
    obs_rec = ra[4]["observations"]
    rows = np.unique(np.concatenate([np.arange(0, n, 16), np.arange(n - 32 * 16, n)]))
    check_values(ra[4]["values"], [[o[t] for o in obs_rec] for t in range(2)], critic, nw.obs_dims, rows=rows)
    check_values(ra[4]["final_values"][None], [list(ra[0])], critic, nw.obs_dims, rows=rows)


@pytest.mark.parametrize("tanh,fn,episodes", [(False, True, False), (True, False, False), (True, True, True)])
def test_on_simple_local_and_centralized_critics_are_bit_identical(tanh, fn, episodes):
    """one agent: obs = share_obs, so the same critic gives the same bits through either kernel"""
    env_a, env_b = twins("simple", 1031)
    nw = env_a.world.native
    pols = make_mappo_actors(nw.obs_dims, nw.act_dims, tanh, fn)
    critic = make_critic(nw.obs_dims, tanh, fn)
    kw = dict(explore_seed=5, action_mode="categorical", episode_length=3 if episodes else None, **RECORDS)
    ra = env_a.rollout_policy(pols, 6, critic=critic, centralized_critic=False, **kw)
    rb = env_b.rollout_policy(pols, 6, critic=critic, **kw)
    compare_outputs(ra, rb, env_a, env_b)
    assert torch.equal(ra[4]["values"], rb[4]["values"]) and torch.equal(ra[4]["final_values"], rb[4]["final_values"])


@pytest.mark.parametrize("tag,mode", [("simple_spread_n3", "shared"), ("simple_spread_n3", "per_agent"),
                                      ("simple_tag", "per_agent"), ("simple_spread_n6", "shared")])
def test_episode_form_equals_the_loop(tag, mode):
    E, L = 3, 4
    n = size(tag, 2, episodes=True, count=count_of(tag, mode))
    env_a, env_b = twins(tag, n)
    env_c = twins(tag, n)[0]
    nw = env_a.world.native
    pols = make_mappo_actors(nw.obs_dims, nw.act_dims, True, True)
    critic = make_local_critics(nw.obs_dims, mode, True, True)
    kw = dict(episode_length=L, explore_seed=21, **RECORDS)
    ra = env_a.rollout_policy(pols, E * L, critic=critic, **LOCAL, **kw)
    rb = env_b.rollout_policy(pols, E * L, action_mode="categorical", **kw)
    compare_outputs(ra, rb, env_a, env_b, keys=("actions", "observations", "final_observations"))
    values, final = ra[4]["values"], ra[4]["final_values"]
    fin = ra[4]["final_observations"]
    check_values(final, [[f[e] for f in fin] for e in range(E)], critic, nw.obs_dims)
    lv, lf = [], []
    for _ in range(E):
        ex = env_c.rollout_policy(pols, L, explore_seed=21, critic=critic, **LOCAL, **RECORDS)[4]
        lv.append(ex["values"])
        lf.append(ex["final_values"])
        env_c.reset()
    torch.cuda.synchronize()
    assert torch.equal(values, torch.cat(lv)) and torch.equal(final, torch.stack(lf))


def test_refusals_leave_state_and_epochs_unchanged():
    from multiagent_particle_envs_b200._lib import MpeError
    for tag, mode in (("simple_tag_4v2", "per_agent"), ("simple_tag_6v2", "per_agent"), ("simple_spread_n5", "per_agent"),
                      ("simple_spread_n6", "per_agent")):
        env = make_product_env(tag, num_envs=64, seed=9)
        env.reset()
        before, epoch = state(env), env.world.native.epoch
        nw = env.world.native
        pols = make_mappo_actors(nw.obs_dims, nw.act_dims, False, True)
        critic = make_local_critics(nw.obs_dims, mode, False, True)
        for kw in ({}, {"episode_length": 2}):
            with pytest.raises(MpeError, match="no compiled"):
                env.rollout_policy(pols, 4, explore_seed=1, critic=critic, **LOCAL, **kw)
            torch.cuda.synchronize()
            for x, y in zip(state(env), before):
                assert torch.equal(x, y)
            assert env.world.native.epoch == epoch and env.explore_epoch == 0


# ---- rIPPO: the recurrent local critic ---------------------------------------------------------------------------------
RECURRENT = dict(action_mode="categorical", record_actions=True, per_step_rewards=True, record_log_probs=True,
                 record_rnn_states=True)


def rippo(tag, n, tanh, fn):
    env_a, env_b = twins(tag, n)
    nw = env_a.world.native
    pols = [make_rmappo_actor(nw.obs_dims[0], nw.act_dims[0], tanh, fn)] * env_a.n
    return env_a, env_b, nw, pols, make_rcritic(nw.obs_dims[:1], tanh, fn)


@pytest.mark.parametrize("tag", ["simple_spread_n3", "simple_spread_n6", "simple_reference"])
@pytest.mark.parametrize("tanh,explore", [(False, True), (True, False)])
def test_recurrent_local_critic_matches_the_modules(tag, tanh, explore):
    fn = explore != tanh
    n, T = 3001, 25
    env_a, env_b, nw, pols, critic = rippo(tag, n, tanh, fn)
    A = env_a.n
    g = torch.Generator(device="cuda").manual_seed(3)
    h0 = torch.tanh(torch.randn(A, n, H, device="cuda", generator=g))
    kw = dict(explore_seed=0x5EED if explore else None, **RECURRENT)
    ra = env_a.rollout_policy(pols, T, critic=critic, critic_rnn_states=h0, record_critic_rnn_states=True,
                              record_observations=True, centralized_critic=False, **kw)
    rb = env_b.rollout_policy(pols, T, record_observations=True, **kw)
    torch.cuda.synchronize()
    for key in ("rewards", "log_probs", "rnn_states", "final_rnn_states"):
        assert torch.equal(ra[4][key], rb[4][key]), key
    for x, y in zip(state(env_a), state(env_b)):
        assert torch.equal(x, y)
    ex = ra[4]
    assert tuple(ex["values"].shape) == (T, A, n) and tuple(ex["final_critic_rnn_states"].shape) == (A, n, H)
    assert tuple(ex["critic_rnn_states"].shape) == (T, A, n, H)
    assert torch.equal(ex["critic_rnn_states"][0], h0)
    rows = np.r_[0:512, n - 512:n]
    loose = 0.0
    for k in range(A):
        x = ex["observations"][k].cpu().numpy()[:, rows].astype(np.float64)
        xf = ra[0][k].cpu().numpy()[rows][None].astype(np.float64)
        mv, mf, _ = module_rollout(critic, x, xf, h0[k].cpu().numpy()[rows])
        loose = max(loose, float(np.abs(ex["values"][:, k].cpu().numpy()[:, rows] - mv).max()),
                    float(np.abs(ex["final_values"][k].cpu().numpy()[rows] - mf[0]).max()))
    assert loose <= LOOSE, loose
    print("\nrecurrent local critic %s tanh=%s feature_norm=%s: within %.2e of the modules run free over T = %d"
          % (tag, tanh, fn, loose, T))


def test_recurrent_local_hidden_states_carry_over_and_calls_are_deterministic():
    """greedy, so that a split call takes the same trajectory: 5 + 5 steps continuing from the final states equal one
    call of 10; two identical calls give identical bits"""
    env_a, env_b, nw, pols, critic = rippo("simple_spread_n3", 2049, False, True)
    env_c = twins("simple_spread_n3", 2049)[0]
    kw = dict(critic=critic, centralized_critic=False, **RECURRENT)
    whole = env_a.rollout_policy(pols, 10, **kw)[4]
    again = env_c.rollout_policy(pols, 10, **kw)[4]
    a = env_b.rollout_policy(pols, 5, **kw)[4]
    b = env_b.rollout_policy(pols, 5, rnn_states=a["final_rnn_states"], critic_rnn_states=a["final_critic_rnn_states"],
                             **kw)[4]
    torch.cuda.synchronize()
    assert torch.equal(whole["values"], again["values"])
    assert torch.equal(whole["final_critic_rnn_states"], again["final_critic_rnn_states"])
    assert torch.equal(whole["values"], torch.cat([a["values"], b["values"]]))
    assert torch.equal(whole["final_values"], b["final_values"])
    assert torch.equal(whole["final_critic_rnn_states"], b["final_critic_rnn_states"])


def test_recurrent_local_episodes_equal_the_loop():
    E, L = 3, 4
    env_a, _, nw, pols, critic = rippo("simple_spread_n3", 1500, True, True)
    env_c = twins("simple_spread_n3", 1500)[0]
    kw = dict(critic=critic, centralized_critic=False, explore_seed=8, **RECURRENT)
    ex = env_a.rollout_policy(pols, E * L, episode_length=L, **kw)[4]
    lv, lf, lh = [], [], []
    for _ in range(E):
        r = env_c.rollout_policy(pols, L, **kw)[4]
        lv.append(r["values"])
        lf.append(r["final_values"])
        lh.append(r["final_critic_rnn_states"])
        env_c.reset()
    torch.cuda.synchronize()
    assert torch.equal(ex["values"], torch.cat(lv)) and torch.equal(ex["final_values"], torch.stack(lf))
    assert torch.equal(ex["final_critic_rnn_states"], lh[-1])


@pytest.mark.parametrize("episodes", [False, True])
def test_on_simple_the_recurrent_local_critic_equals_the_centralized_one(episodes):
    env_a, env_b, nw, pols, critic = rippo("simple", 1031, True, True)
    kw = dict(critic=critic, explore_seed=2, record_critic_rnn_states=True, episode_length=4 if episodes else None,
              **RECURRENT)
    ra = env_a.rollout_policy(pols, 8, centralized_critic=False, **kw)[4]
    rb = env_b.rollout_policy(pols, 8, **kw)[4]
    torch.cuda.synchronize()
    assert torch.equal(ra["values"], rb["values"]) and torch.equal(ra["final_values"], rb["final_values"])
    assert torch.equal(ra["final_critic_rnn_states"][0], rb["final_critic_rnn_states"])
    assert torch.equal(ra["critic_rnn_states"][:, 0], rb["critic_rnn_states"])


def test_gae_over_ippo_values_with_a_per_agent_value_norm():
    tag = "simple_spread_n3"
    n = size(tag, 2, count=3)
    env, _ = twins(tag, n)
    nw = env.world.native
    pols = make_mappo_actors(nw.obs_dims, nw.act_dims, False, True)
    critic = make_local_critics(nw.obs_dims, "per_agent", False, True)
    ex = env.rollout_policy(pols, 25, explore_seed=7, critic=critic, **LOCAL, **RECORDS)[4]
    vn = torch.tensor([[0.3, 1.7], [-0.2, 0.6], [0.1, 1.1]], dtype=torch.float32, device="cuda")
    ret, adv, _ = env.compute_gae(ex["rewards"], ex["values"], ex["final_values"], value_norm=vn)
    want_ret, want_adv, _ = gae_mirror(ex["rewards"].cpu().numpy(), ex["values"].cpu().numpy(),
                                       ex["final_values"].cpu().numpy()[None], 0.99, 0.95, value_norm=vn.cpu().numpy())
    assert np.array_equal(ret.cpu().numpy(), want_ret) and np.array_equal(adv.cpu().numpy(), want_adv)
