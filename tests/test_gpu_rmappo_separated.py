"""env.rollout_policy([speaker, listener], T, action_mode="categorical", critic=[critic0, critic1]) on
simple_speaker_listener: rMAPPO's separated runner, every agent's own recurrent actor (restaged into one shared-memory
slot at each agent's turn) and its own recurrent critic (mpe_rollout_policy_gru_separated[_episodes],
mpe_critic_gru_separated).  ReLU and tanh, exploring and greedy, the input LayerNorm on for half of the cases, at a
ragged size whose last block has idle warps and whose last warp is partial, and at a multi-wave 65 553 worlds: replay of
the recorded indices through a twin env, bit for bit; each agent's h' teacher-forced on the records within the written
bound; every pick and log-probability explained; weight isolation (the speaker does not depend on the listener's
weights); determinism; carrying both hidden states across calls; the episode form against its loop; the critics
against the call without them, the written value bound and the unfolded float64 critics; GAE with a per-agent
ValueNorm on the outputs; the refusals."""
import numpy as np
import pytest

from gae_helpers import gae_mirror
from helpers import device_sms, launch_shape, make_product_env, regime_size
from mappo_helpers import FEATURE_NORM, TANH
from mlp_categorical_helpers import bounds, log_softmax_at, one_hot_torch
from mlp_helpers import gumbel_noise
from mlp_programs import state, twins
from rcritic_helpers import LOOSE, make_rcritic, module_rollout, value_bound
from rmappo_helpers import H, RecurrentModel, explain_head_mismatches, make_rmappo_actor, module_step

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

TAG = "simple_speaker_listener"
WARPS = 8
LOGP_FLIP_SLACK = 1e-3
TIGHT_SHARE = 0.95
RECORDS = dict(record_actions=True, per_step_rewards=True, record_observations=True, record_log_probs=True,
               record_rnn_states=True)
SEGMENTS = [[3], [5]]       # the speaker utters 1 of 3 symbols, the listener moves
CHECK_ROWS = 1024           # worlds checked against the float64 models: the first and the last ones


def ragged(base=None):
    """8-warp blocks, a last block with idle warps and a last warp of 17 worlds"""
    sms = device_sms()
    n = regime_size("mlp", sms, WARPS, cap=WARPS, base=base)
    wpb, blocks, partial, last = launch_shape("mlp", n, sms, WARPS)
    assert wpb == WARPS and partial and last == 17
    assert (n + 31) // 32 % WARPS != 0            # the last block has warps without worlds
    return n


def actors(nw, tanh, fn, seeds=(3, 4), eps=1e-5):
    return [make_rmappo_actor(od, ad, tanh, fn, seed=s, eps=eps) for od, ad, s in zip(nw.obs_dims, nw.act_dims, seeds)]


def critics(nw, tanh, fn, seeds=(7, 8)):
    return [make_rcritic(nw.obs_dims, tanh, fn, seed=s) for s in seeds]


def model_of(actor, od, ad):
    from multiagent_particle_envs_b200.environment import rmappo_actor_params
    params, tanh, fn, eps = rmappo_actor_params([actor], [od], [ad])
    net = ((FEATURE_NORM if fn else 0) | (TANH if tanh else 0), eps)
    return RecurrentModel([t.to(torch.float32).cpu().numpy() for t in params], net)


def critic_model(critic, obs_dims):
    from multiagent_particle_envs_b200.environment import rmappo_critic_params
    params, tanh, fn, eps = rmappo_critic_params(critic, obs_dims)
    net = ((FEATURE_NORM if fn else 0) | (TANH if tanh else 0), eps)
    return RecurrentModel([t.to(torch.float32).cpu().numpy() for t in params], net)


def observe(env):
    nw = env.world.native
    return [o.clone() for o in nw.observe(out=nw.new_outputs(), flags=env._flags()).obs]


def check_rows(n):
    return np.arange(n) if n <= CHECK_ROWS else np.r_[0:CHECK_ROWS // 2, n - CHECK_ROWS // 2:n]


def same(a, b):
    torch.cuda.synchronize()
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def check_replay_and_numerics(n, T, explore, tanh, fn):
    env_a, env_b = twins(TAG, n)
    na = env_a.world.native
    A = env_a.n
    pols = actors(na, tanh, fn)
    models = [model_of(p, od, ad) for p, od, ad in zip(pols, na.obs_dims, na.act_dims)]
    seed = 0x1234_5678_9ABC if explore else None
    obs_b = observe(env_b)
    obs_r, rew_r, done_r, _, ex = env_a.rollout_policy(pols, T, explore_seed=seed, action_mode="categorical", **RECORDS)
    idx, logp, rew_steps, obs_rec = ex["actions"], ex["log_probs"], ex["rewards"], ex["observations"]
    hrec, hfin = ex["rnn_states"], ex["final_rnn_states"]
    assert tuple(hrec.shape) == (T, A, n, H) and tuple(hfin.shape) == (A, n, H)
    assert not bool(hrec[0].any())
    rows = check_rows(n)
    rew_sum = torch.zeros(A, n, device="cuda")
    flips = gaps = 0
    lmax = 0.0
    tight_in = total = 0
    for t in range(T):
        for i in range(A):
            assert torch.equal(obs_rec[i][t], obs_b[i]), (t, i)
            model = models[i]
            o = obs_b[i].cpu().numpy()[rows]
            h = hrec[t, i].cpu().numpy()[rows].astype(np.float64)
            hk = (hrec[t + 1, i] if t + 1 < T else hfin[i]).cpu().numpy()[rows].astype(np.float64)
            d = np.abs(hk - model.gru(model.base(o), h))
            loose = model.h_bound(o, h, True)
            assert (d <= loose).all(), (t, i, float((d - loose).max()))
            tight_in += int((d <= model.h_bound(o, h, False)).sum())
            total += d.size
            g = gumbel_noise(seed, 0, rows, t, i, A, n_logits=na.act_dims[i], stride=2) if explore else 0.0
            k = idx[i][t].cpu().numpy()[rows]
            lp = logp[t, i].cpu().numpy()[rows].astype(np.float64)
            f, gp = explain_head_mismatches(k, lp, hk, model, SEGMENTS[i], noise=g)
            flips, gaps = flips + f, gaps + gp
            z64, _ = module_step(pols[i], o, h)
            err = np.abs(lp - log_softmax_at(z64, k, SEGMENTS[i]))
            lmax = max(lmax, float(err.max()))
            dz = np.abs(model.logits(hk) - z64)
            bound = sum(2.0 * dz[:, a:b].max(-1) for a, b in bounds(SEGMENTS[i])) + LOGP_FLIP_SLACK
            assert (err <= bound).all(), (t, i, float((err - bound).max()))
        obs_b, rew_s, _, _ = env_b.step([one_hot_torch(k[t], s) for k, s in zip(idx, SEGMENTS)])
        rew_sum += torch.stack(list(rew_s))
        assert torch.equal(rew_steps[t], torch.stack(list(rew_s))), t
    torch.cuda.synchronize()
    same(state(env_a), state(env_b))
    same(obs_r, obs_b)
    assert torch.equal(torch.stack(list(rew_r)), rew_sum)
    assert not any(bool(x.any()) for x in done_r)
    assert env_a.explore_epoch == (1 if explore else 0)
    share = tight_in / total
    print("\nseparated rmappo tanh=%s feature_norm=%s n=%d explore=%s: h' within the flip-free bound for %.4f of "
          "entries, all within the bound with flips; %d rows explained by TF32 flips of LN(h'), %d by the Gumbel gap; "
          "log-probabilities within %.3e of the unfolded float64 modules" % (tanh, fn, n, explore, share, flips, gaps, lmax))
    assert share >= TIGHT_SHARE, share


@pytest.mark.parametrize("tanh", [False, True])
@pytest.mark.parametrize("explore", [True, False])
def test_separated_replay_and_numerics(tanh, explore):
    """the input LayerNorm is on for (ReLU, exploring) and (tanh, greedy)"""
    check_replay_and_numerics(ragged(), 3, explore, tanh, fn=(explore != tanh))


def test_separated_replay_multi_wave():
    """65 536 worlds plus a ragged tail: more blocks than SMs, a last block of one warp"""
    check_replay_and_numerics(ragged(base=65536), 2, True, False, fn=True)


def test_weight_isolation():
    """The speaker observes the goal colour only, so its trajectory does not depend on the listener: with only the
    listener's weights changed, the speaker's picks, log-probabilities and h are bit-identical and the listener's are
    not.  A restaging race or a wrong slot would mix them."""
    n = ragged()
    env_a, env_b = twins(TAG, n)
    nw = env_a.world.native
    speaker, listener = actors(nw, True, True)
    other = actors(nw, True, True, seeds=(3, 11))[1]
    kw = dict(explore_seed=77, action_mode="categorical", **RECORDS)
    ra = env_a.rollout_policy([speaker, listener], 8, **kw)[4]
    rb = env_b.rollout_policy([speaker, other], 8, **kw)[4]
    torch.cuda.synchronize()
    assert torch.equal(ra["actions"][0], rb["actions"][0])
    assert torch.equal(ra["log_probs"][:, 0], rb["log_probs"][:, 0])
    assert torch.equal(ra["rnn_states"][:, 0], rb["rnn_states"][:, 0])
    assert torch.equal(ra["final_rnn_states"][0], rb["final_rnn_states"][0])
    assert not torch.equal(ra["log_probs"][:, 1], rb["log_probs"][:, 1])
    assert not torch.equal(ra["rnn_states"][1:, 1], rb["rnn_states"][1:, 1])


def test_identical_calls_are_identical():
    n = ragged()
    env_a, env_b = twins(TAG, n)
    nw = env_a.world.native
    pols, crit = actors(nw, False, True), critics(nw, False, True)
    for kw in ({}, {"episode_length": 5}):
        args = dict(explore_seed=4, action_mode="categorical", critic=crit, record_critic_rnn_states=True, **kw,
                    **RECORDS)
        ra = env_a.rollout_policy(pols, 10, **args)
        rb = env_b.rollout_policy(pols, 10, **args)
        torch.cuda.synchronize()
        for key in ("rewards", "log_probs", "rnn_states", "final_rnn_states", "values", "final_values",
                    "critic_rnn_states", "final_critic_rnn_states"):
            assert torch.equal(ra[4][key], rb[4][key]), key
        same(ra[4]["actions"], rb[4]["actions"])
        same(ra[0], rb[0])
        same(state(env_a), state(env_b))


def test_hidden_states_carry_over_between_calls():
    """two greedy calls of T1 and T2 carrying rnn_states and critic_rnn_states == one call of T1 + T2, bit for bit"""
    n, T1, T2 = ragged(), 12, 13
    env_a, env_b = twins(TAG, n)
    nw = env_a.world.native
    pols, crit = actors(nw, True, False), critics(nw, True, False)
    kw = dict(action_mode="categorical", critic=crit, record_critic_rnn_states=True, **RECORDS)
    ra = env_a.rollout_policy(pols, T1 + T2, **kw)[4]
    rb1 = env_b.rollout_policy(pols, T1, **kw)[4]
    h, hc = rb1["final_rnn_states"].clone(), rb1["final_critic_rnn_states"].clone()
    rb2 = env_b.rollout_policy(pols, T2, rnn_states=h, critic_rnn_states=hc, **kw)[4]
    torch.cuda.synchronize()
    assert torch.equal(h, rb1["final_rnn_states"]) and torch.equal(hc, rb1["final_critic_rnn_states"])   # never written
    assert tuple(rb2["final_critic_rnn_states"].shape) == (2, n, H)
    assert tuple(rb2["critic_rnn_states"].shape) == (T2, 2, n, H)
    for key in ("values", "critic_rnn_states", "rnn_states", "log_probs", "rewards"):
        assert torch.equal(ra[key], torch.cat([rb1[key], rb2[key]])), key
    for key in ("final_values", "final_critic_rnn_states", "final_rnn_states"):
        assert torch.equal(ra[key], rb2[key]), key
    assert torch.equal(rb2["rnn_states"][0], h) and torch.equal(rb2["critic_rnn_states"][0], hc)
    same(state(env_a), state(env_b))


KEYS = ("rewards", "log_probs", "rnn_states", "values", "critic_rnn_states")
LIST_KEYS = ("actions", "observations")


@pytest.mark.parametrize("E,L,explore,tanh,fn", [(3, 4, True, True, True), (2, 3, False, False, False)])
def test_episodes_equal_the_loop(E, L, explore, tanh, fn):
    n = ragged()
    env_a, env_b = twins(TAG, n)
    nw = env_a.world.native
    pols, crit = actors(nw, tanh, fn), critics(nw, tanh, fn)
    seed = 21 if explore else None
    kw = dict(explore_seed=seed, action_mode="categorical", critic=crit, record_critic_rnn_states=True, **RECORDS)
    epoch = nw.epoch
    obs, ret, done, _, ex = env_a.rollout_policy(pols, E * L, episode_length=L, **kw)
    parts = {k: [] for k in KEYS + LIST_KEYS}
    finals, fvals, rets = [], [], []
    for _ in range(E):
        obs_e, rew_e, _, _, exl = env_b.rollout_policy(pols, L, **kw)
        for k in parts:
            parts[k].append(exl[k])
        finals.append(obs_e)
        fvals.append(exl["final_values"])
        rets.append(rew_e)
        last = exl
        obs_b = env_b.reset()
    torch.cuda.synchronize()
    assert tuple(ex["final_values"].shape) == (E, 2, n)
    for e in range(E):
        assert not bool(ex["rnn_states"][e * L].any()) and not bool(ex["critic_rnn_states"][e * L].any()), e
    for k in KEYS:
        assert torch.equal(ex[k], torch.cat(parts[k])), k
    for k in LIST_KEYS:
        for i in range(2):
            assert torch.equal(ex[k][i], torch.cat([p[i] for p in parts[k]])), (k, i)
    assert torch.equal(ex["final_values"], torch.stack(fvals))
    for k in ("final_rnn_states", "final_critic_rnn_states"):
        assert torch.equal(ex[k], last[k]), k
    for i in range(2):
        assert torch.equal(ex["final_observations"][i], torch.stack([f[i] for f in finals])), i
        assert torch.equal(ret[i], torch.stack([r[i] for r in rets])), i
        assert torch.equal(obs[i], obs_b[i]), i
        assert not bool(done[i].any())
    same(state(env_a), state(env_b))
    assert nw.epoch == env_b.world.native.epoch == epoch + E


@pytest.mark.parametrize("tanh,explore", [(False, True), (True, False)])
def test_critics_change_nothing_and_match_the_models(tanh, explore):
    """per-agent critics: every other output bit-identical to the call without them; critic k's h' teacher-forced on
    its own h_t and share_obs_t within the bound with flips; its values within value_bound given its h', and within
    LOOSE of the unfolded float64 critic run free from its h0; GAE with a per-agent ValueNorm equals the mirror"""
    fn = explore != tanh
    T = 25
    n = ragged(base=65536) if explore else ragged()
    env_a, env_b = twins(TAG, n)
    nw = env_a.world.native
    pols, crit = actors(nw, tanh, fn), critics(nw, tanh, fn)
    g = torch.Generator(device="cuda").manual_seed(3)
    h0 = torch.tanh(torch.randn(2, n, H, device="cuda", generator=g))
    h0_in = h0.clone()
    kw = dict(explore_seed=0x5EED if explore else None, action_mode="categorical", **RECORDS)
    ra = env_a.rollout_policy(pols, T, critic=crit, critic_rnn_states=h0, record_critic_rnn_states=True, **kw)
    rb = env_b.rollout_policy(pols, T, **kw)
    same(ra[0] + ra[1] + ra[2], rb[0] + rb[1] + rb[2])
    for key in ("rewards", "log_probs", "rnn_states", "final_rnn_states"):
        assert torch.equal(ra[4][key], rb[4][key]), key
    same(ra[4]["actions"], rb[4]["actions"])
    same(ra[4]["observations"], rb[4]["observations"])
    same(state(env_a), state(env_b))
    assert nw.epoch == env_b.world.native.epoch and env_a.explore_epoch == env_b.explore_epoch
    assert torch.equal(h0, h0_in)
    ex = ra[4]
    values, final, hrec, hfin = ex["values"], ex["final_values"], ex["critic_rnn_states"], ex["final_critic_rnn_states"]
    assert tuple(values.shape) == (T, 2, n) and tuple(final.shape) == (2, n)
    assert tuple(hrec.shape) == (T, 2, n, H) and tuple(hfin.shape) == (2, n, H)
    assert torch.equal(hrec[0], h0)
    assert not torch.equal(values[:, 0], values[:, 1])
    rows = check_rows(n)
    x = np.concatenate([o.cpu().numpy()[:, rows] for o in rb[4]["observations"]], -1).astype(np.float64)
    x_final = np.concatenate([o.cpu().numpy()[rows] for o in ra[0]], -1).astype(np.float64)[None]
    loose = 0.0
    for k in range(2):
        model = critic_model(crit[k], nw.obs_dims)
        hr = hrec[:, k].cpu().numpy()[:, rows].astype(np.float64)
        hnext = np.concatenate([hr[1:], hfin[k].cpu().numpy()[rows][None].astype(np.float64)])
        v = values[:, k].cpu().numpy()[:, rows].astype(np.float64)
        for t in range(T):
            err = np.abs(hnext[t] - model.gru(model.base(x[t]), hr[t]))
            bound = model.h_bound(x[t], hr[t], flips=True)
            assert (err <= bound).all(), (k, t, float((err - bound).max()))
            verr = np.abs(v[t] - model.logits(hnext[t])[:, 0])
            vb = value_bound(model, hnext[t])
            assert (verr <= vb).all(), (k, t, float((verr - vb).max()))
        mv, mf, _ = module_rollout(crit[k], x, x_final, h0[k].cpu().numpy()[rows])
        loose = max(loose, float(np.abs(v - mv).max()), float(np.abs(final[k].cpu().numpy()[rows] - mf[0]).max()))
    assert loose <= LOOSE, loose
    print("\nseparated rcritic tanh=%s feature_norm=%s n=%d: values within %.2e of the unfolded float64 critics run "
          "free over T = %d" % (tanh, fn, n, loose, T))
    # ---- GAE over the outputs, one ValueNorm row per agent ----
    vn = torch.tensor([[0.3, 1.7], [-0.2, 0.6]], dtype=torch.float32, device="cuda")
    ret, adv, _ = env_a.compute_gae(ex["rewards"], values, final, value_norm=vn)
    want_ret, want_adv, _ = gae_mirror(ex["rewards"].cpu().numpy(), values.cpu().numpy(), final.cpu().numpy()[None],
                                       0.99, 0.95, value_norm=vn.cpu().numpy())
    assert np.array_equal(ret.cpu().numpy(), want_ret) and np.array_equal(adv.cpu().numpy(), want_adv)


def test_refusals_leave_state_and_epochs_unchanged():
    from multiagent_particle_envs_b200._lib import MpeError
    env = make_product_env(TAG, num_envs=64, seed=9)
    env.reset()
    nw = env.world.native
    pols, crit = actors(nw, False, True), critics(nw, False, True)
    before, epoch = state(env), nw.epoch

    def unchanged(e, b, ep):
        torch.cuda.synchronize()
        for x, y in zip(state(e), b):
            assert torch.equal(x, y)
        assert e.world.native.epoch == ep and e.explore_epoch == 0

    cat = dict(action_mode="categorical", explore_seed=1, record_log_probs=True)
    refusals = [
        (ValueError, "agent 0's recurrent actor", dict(policies=pols[::-1])),
        (ValueError, "same activation", dict(policies=[pols[0], actors(nw, True, True)[1]])),
        (ValueError, "list of 2 recurrent critics", dict(critic=crit[0])),
        (ValueError, "list of 2 recurrent critics", dict(critic=crit + crit[:1])),
        (ValueError, "critic must use", dict(critic=critics(nw, True, True))),
        (ValueError, "critic_rnn_states", dict(critic=crit, critic_rnn_states=torch.zeros(64, H, device="cuda"))),
        (ValueError, "critic_rnn_states", dict(critic=crit, critic_rnn_states=torch.zeros(2, 64, H))),
        (ValueError, "rnn_states", dict(rnn_states=torch.zeros(2, 64, 32, device="cuda"))),
        (ValueError, "episode_length", dict(episode_length=2, rnn_states=torch.zeros(2, 64, H, device="cuda"))),
        (MpeError, "no compiled", dict(policies=[pols[1]] * 2)),               # one shared tuple: no such kernel
    ]
    for exc, match, kw in refusals:
        with pytest.raises(exc, match=match):
            env.rollout_policy(kw.pop("policies", pols), 4, **cat, **kw)
        unchanged(env, before, epoch)
    spread = make_product_env("simple_spread_n3", num_envs=64, seed=9)   # distinct tuples on a homogeneous program
    spread.reset()
    sbefore, sepoch = state(spread), spread.world.native.epoch
    a = make_rmappo_actor(18, 5, False, True)
    c = make_rcritic([18] * 3, False, True)
    with pytest.raises(NotImplementedError, match="shared"):
        spread.rollout_policy([a, tuple(list(a)), a], 4, **cat)
    unchanged(spread, sbefore, sepoch)
    with pytest.raises(NotImplementedError, match="distinct"):
        spread.rollout_policy([a] * 3, 4, critic=[c, tuple(list(c)), c], **cat)
    unchanged(spread, sbefore, sepoch)
