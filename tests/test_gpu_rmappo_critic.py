"""env.rollout_policy(rmappo_actors, T, action_mode="categorical", critic=(base, gru, norm, v_out)) (mpe_critic_gru):
rMAPPO's recurrent centralized critic, run after the recurrent actor's rollout over its observation records.  For the
seven programs of the recurrent actor, ReLU and tanh, exploring and greedy, the input LayerNorm on for half of the
cases and two cases at a ragged 65 553 worlds: every other output, the state and both epochs bit-identical to the same
call without a critic; the critic's recorded h starting from h0 bitwise; every h' teacher-forced on the kernel's own
h_t and share_obs_t within RecurrentModel.h_bound(flips=True); every value, given the kernel's h', within value_bound;
every value within LOOSE of the unfolded float64 modules run free from h0; carrying both hidden states from one call
to the next; the episode form against its loop; determinism; the refusals."""
import numpy as np
import pytest

from helpers import make_product_env
from mappo_helpers import FEATURE_NORM, TANH
from mlp_programs import state, twins
from rcritic_helpers import H, LOOSE, RCRITIC_PROGRAMS, RecurrentModel, make_rcritic, module_rollout, value_bound
from rmappo_helpers import make_rmappo_actor

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

RECORDS = dict(record_actions=True, per_step_rewards=True, record_log_probs=True, record_rnn_states=True)
T = 25
CASES = [(tag, tanh, explore) for tag in RCRITIC_PROGRAMS for tanh in (False, True) for explore in (True, False)]
RAGGED = {("simple_spread_n3", False, True): 65553, ("simple_spread_n6", True, False): 65553}
CHECK_ROWS = 1024          # worlds checked against the float64 models: the first and the last ones


def model_of(critic, nw):
    from multiagent_particle_envs_b200.environment import rmappo_critic_params
    params, tanh, fn, eps = rmappo_critic_params(critic, nw.obs_dims)
    net = ((FEATURE_NORM if fn else 0) | (TANH if tanh else 0), eps)
    return RecurrentModel([t.to(torch.float32).cpu().numpy() for t in params], net)


def share(obs_list, rows):
    """share_obs of the selected worlds: agent observations [..., N, obs_dim_i] -> [..., rows, D] in float64"""
    return np.concatenate([o.cpu().numpy()[..., rows, :] for o in obs_list], -1).astype(np.float64)


def same(a, b):
    torch.cuda.synchronize()
    for x, y in zip(a, b):
        assert torch.equal(x, y)


@pytest.mark.parametrize("tag,tanh,explore", CASES)
def test_rcritic_changes_nothing_and_matches_the_models(tag, tanh, explore):
    fn = explore != tanh
    n = RAGGED.get((tag, tanh, explore), 300)
    env_a, env_b = twins(tag, n)
    nw = env_a.world.native
    A = env_a.n
    pols = [make_rmappo_actor(nw.obs_dims[0], nw.act_dims[0], tanh, fn)] * A
    critic = make_rcritic(nw.obs_dims, tanh, fn)
    g = torch.Generator(device="cuda").manual_seed(3)
    h0 = torch.tanh(torch.randn(n, H, device="cuda", generator=g))
    h0_in = h0.clone()
    kw = dict(explore_seed=0x5EED if explore else None, action_mode="categorical", **RECORDS)
    ra = env_a.rollout_policy(pols, T, critic=critic, critic_rnn_states=h0, record_critic_rnn_states=True, **kw)
    rb = env_b.rollout_policy(pols, T, record_observations=True, **kw)
    # ---- everything but the critic's outputs is the call without a critic, bit for bit ----
    same(ra[0] + ra[1] + ra[2], rb[0] + rb[1] + rb[2])
    for key in ("rewards", "log_probs", "rnn_states", "final_rnn_states"):
        assert torch.equal(ra[4][key], rb[4][key]), key
    same(ra[4]["actions"], rb[4]["actions"])
    assert ra[4]["observations"] is None                     # the scratch records stay internal
    same(state(env_a), state(env_b))
    assert nw.epoch == env_b.world.native.epoch and env_a.explore_epoch == env_b.explore_epoch
    assert torch.equal(h0, h0_in)                            # the input state is never written
    ex = ra[4]
    values, final, hrec, hfin = ex["values"], ex["final_values"], ex["critic_rnn_states"], ex["final_critic_rnn_states"]
    assert tuple(values.shape) == (T, A, n) and tuple(final.shape) == (A, n)
    assert tuple(hrec.shape) == (T, n, H) and tuple(hfin.shape) == (n, H)
    assert all(t.dtype == torch.float32 for t in (values, final, hrec, hfin))
    assert torch.equal(hrec[0], h0)
    for i in range(1, A):                                    # the shared value, written for every agent
        assert torch.equal(values[:, i], values[:, 0]) and torch.equal(final[i], final[0])
    # ---- teacher-forced on the kernel's own h_t and share_obs_t ----
    model = model_of(critic, nw)
    rows = np.arange(n) if n <= CHECK_ROWS else np.r_[0:CHECK_ROWS // 2, n - CHECK_ROWS // 2:n]
    x = share(rb[4]["observations"], rows)                   # [T, r, D]
    hr = hrec.cpu().numpy()[:, rows].astype(np.float64)
    hnext = np.concatenate([hr[1:], hfin.cpu().numpy()[rows][None].astype(np.float64)])
    v = values[:, 0].cpu().numpy()[:, rows].astype(np.float64)
    tight, total = 0, 0
    for t in range(T):
        want = model.gru(model.base(x[t]), hr[t])
        err = np.abs(hnext[t] - want)
        tight += int((err <= model.h_bound(x[t], hr[t], flips=False)).sum())
        total += err.size
        bound = model.h_bound(x[t], hr[t], flips=True)
        assert (err <= bound).all(), (t, float((err - bound).max()))
        verr = np.abs(v[t] - model.logits(hnext[t])[:, 0])
        vb = value_bound(model, hnext[t])
        assert (verr <= vb).all(), (t, float((verr - vb).max()))
    # ---- against the unfolded float64 modules, run free from h0 ----
    mv, mf, _ = module_rollout(critic, x, share(list(ra[0]), rows)[None], h0.cpu().numpy()[rows])
    loose = max(float(np.abs(v - mv).max()), float(np.abs(final[0].cpu().numpy()[rows] - mf[0]).max()))
    assert loose <= LOOSE, loose
    print("\nrcritic %s tanh=%s feature_norm=%s n=%d: %.2f %% of h' within the flip-free bound; values within %.2e of "
          "the unfolded float64 critic run free over T = %d" % (tag, tanh, fn, n, 100.0 * tight / total, loose, T))


@pytest.mark.parametrize("tag", ["simple_spread_n3", "simple_reference"])
def test_hidden_states_carry_over_between_calls(tag):
    """two greedy calls of T1 and T2 carrying rnn_states and critic_rnn_states == one call of T1 + T2, bit for bit"""
    T1, T2 = 12, 13
    env_a, env_b = twins(tag, 300)
    nw = env_a.world.native
    pols = [make_rmappo_actor(nw.obs_dims[0], nw.act_dims[0], False, True)] * env_a.n
    critic = make_rcritic(nw.obs_dims, False, True)
    kw = dict(action_mode="categorical", critic=critic, record_critic_rnn_states=True, **RECORDS)
    ra = env_a.rollout_policy(pols, T1 + T2, **kw)
    rb1 = env_b.rollout_policy(pols, T1, **kw)
    rb2 = env_b.rollout_policy(pols, T2, rnn_states=rb1[4]["final_rnn_states"],
                               critic_rnn_states=rb1[4]["final_critic_rnn_states"], **kw)
    torch.cuda.synchronize()
    for key in ("values", "critic_rnn_states", "rnn_states", "log_probs"):
        assert torch.equal(ra[4][key], torch.cat([rb1[4][key], rb2[4][key]])), key
    for key in ("final_values", "final_critic_rnn_states", "final_rnn_states"):
        assert torch.equal(ra[4][key], rb2[4][key]), key
    same(state(env_a), state(env_b))


def rcritic_loop(env, pols, critic, E, L, seed):
    parts = {k: [] for k in ("values", "critic_rnn_states", "log_probs")}
    finals = []
    for _ in range(E):
        ex = env.rollout_policy(pols, L, explore_seed=seed, action_mode="categorical", critic=critic,
                                record_critic_rnn_states=True, **RECORDS)[4]
        for k in parts:
            parts[k].append(ex[k])
        finals.append(ex["final_values"])
        h = ex["final_critic_rnn_states"]
        env.reset()
    out = {k: torch.cat(v) for k, v in parts.items()}
    out.update(final_values=torch.stack(finals), final_critic_rnn_states=h)
    return out


@pytest.mark.parametrize("tag", RCRITIC_PROGRAMS)
@pytest.mark.parametrize("E,L,explore,tanh,fn", [(3, 4, True, True, True), (2, 3, False, False, False)])
def test_rcritic_episodes_equal_the_loop(tag, E, L, explore, tanh, fn):
    env_a, env_b = twins(tag, 300)
    nw = env_a.world.native
    pols = [make_rmappo_actor(nw.obs_dims[0], nw.act_dims[0], tanh, fn)] * env_a.n
    critic = make_rcritic(nw.obs_dims, tanh, fn)
    seed = 21 if explore else None
    ex = env_a.rollout_policy(pols, E * L, episode_length=L, explore_seed=seed, action_mode="categorical", critic=critic,
                              record_critic_rnn_states=True, **RECORDS)[4]
    ref = rcritic_loop(env_b, pols, critic, E, L, seed)
    torch.cuda.synchronize()
    assert tuple(ex["final_values"].shape) == (E, env_a.n, 300) and ex["final_observations"] is None
    for e in range(E):
        assert not bool(ex["critic_rnn_states"][e * L].any()), e          # every episode starts from h = 0
    for key in ("values", "final_values", "critic_rnn_states", "final_critic_rnn_states", "log_probs"):
        assert torch.equal(ex[key], ref[key]), key
    same(state(env_a), state(env_b))


def test_identical_calls_are_identical_and_requested_records_come_back():
    tag = "simple_spread_n4"
    env_a, env_b = twins(tag, 300)
    nw = env_a.world.native
    pols = [make_rmappo_actor(nw.obs_dims[0], nw.act_dims[0], True, True)] * env_a.n
    critic = make_rcritic(nw.obs_dims, True, True)
    for kw in ({}, {"episode_length": 5}):
        args = dict(explore_seed=4, action_mode="categorical", critic=critic, record_observations=True, **kw, **RECORDS)
        ra = env_a.rollout_policy(pols, 10, **args)
        rb = env_b.rollout_policy(pols, 10, **args)
        torch.cuda.synchronize()
        for key in ("values", "final_values", "final_critic_rnn_states"):
            assert torch.equal(ra[4][key], rb[4][key]), key
        assert ra[4]["critic_rnn_states"] is None
        same(ra[4]["observations"], rb[4]["observations"])
        assert all(tuple(o.shape) == (10, 300, od) for o, od in zip(ra[4]["observations"], nw.obs_dims))
        if kw:
            same(ra[4]["final_observations"], rb[4]["final_observations"])


def test_refusals_leave_state_and_epochs_unchanged():
    env = make_product_env("simple_spread_n3", num_envs=64, seed=9)
    env.reset()
    nw = env.world.native
    actor = make_rmappo_actor(18, 5, False, True)
    critic = make_rcritic(nw.obs_dims, False, True)
    before, epoch = state(env), nw.epoch

    def unchanged():
        torch.cuda.synchronize()
        for x, y in zip(state(env), before):
            assert torch.equal(x, y)
        assert nw.epoch == epoch and env.explore_epoch == 0

    cat = dict(action_mode="categorical", explore_seed=1, record_log_probs=True)
    pols = [actor] * 3
    refusals = [
        (NotImplementedError, "distinct", dict(critic=[critic, tuple(list(critic)), critic])),
        (ValueError, "num_layers=1", dict(critic=(critic[0], torch.nn.GRU(64, 64, num_layers=2).cuda(), critic[2],
                                                  critic[3]))),
        (ValueError, "activation", dict(critic=make_rcritic(nw.obs_dims, True, True))),
        (ValueError, "activation", dict(critic=make_rcritic(nw.obs_dims, False, False))),
        (ValueError, "activation", dict(critic=make_rcritic(nw.obs_dims, False, True, eps=1e-3))),
        (ValueError, "episode_length", dict(critic=critic, episode_length=2,
                                            critic_rnn_states=torch.zeros(64, H, device="cuda"))),
        (ValueError, "critic_rnn_states", dict(critic_rnn_states=torch.zeros(64, H, device="cuda"))),
        (ValueError, "critic_rnn_states", dict(record_critic_rnn_states=True)),
    ]
    for h0 in (torch.zeros(64, 32, device="cuda"), torch.zeros(64, H, device="cuda", dtype=torch.float64),
               torch.zeros(64, H), torch.zeros(3, 64, H, device="cuda")):
        refusals.append((ValueError, "critic_rnn_states", dict(critic=critic, critic_rnn_states=h0)))
    for exc, match, kw in refusals:
        with pytest.raises(exc, match=match):
            env.rollout_policy(pols, 4, **cat, **kw)
        unchanged()
