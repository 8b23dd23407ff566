"""env.rollout_policy(..., action_mode="categorical") with MAPPO's recurrent actor (mpe_rollout_policy_gru and its
episode form): one (base, gru, norm, head) tuple shared by every agent, h carried across steps.  Checked for every
program the kernel is built for, with ReLU and tanh, exploring and greedy, the input LayerNorm on for half of the cases:
replay of the recorded indices as one-hot vectors through fused steps of a twin env, bit for bit; every step's h'
teacher-forced on the records against the float64 recipe model under a written bound; every pick and log-probability
against the model evaluated on the kernel's own h', and against the user's unfolded modules; carrying h from one call
to the next; the episode form against its loop; the shared policy; the refusals."""
import numpy as np
import pytest

from helpers import device_sms, launch_shape, make_product_env, regime_size
from mappo_helpers import FEATURE_NORM, TANH
from mlp_categorical_helpers import bounds, log_softmax_at, one_hot_torch
from mlp_helpers import gumbel_noise
from mlp_programs import state, twins
from rmappo_helpers import H, RecurrentModel, explain_head_mismatches, make_rmappo_actor, module_step
from test_cpu_rmappo_actor import GRU_PROGRAMS, GRU_WARPS

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

LOGP_FLIP_SLACK = 1e-3
RECORDS = dict(record_actions=True, per_step_rewards=True, record_observations=True, record_log_probs=True,
               record_rnn_states=True)
# h' within the flip-free bound (RecurrentModel.h_bound(flips=False)) for at least this share of its entries: the rest
# are rows where a TF32 rounding flip of a normalised operand of the base changed x, which the bound with flips covers.
TIGHT_SHARE = 0.95


def segments_of(env):
    d = env.world.native.desc
    return [([5] if d.agent_movable[i] else []) + ([d.dim_c] if not d.agent_silent[i] else []) for i in range(env.n)]


def size(wpb, base=None):
    sms = device_sms()
    n = regime_size("mlp", sms, min(wpb, GRU_WARPS), cap=GRU_WARPS, base=base)
    assert launch_shape("mlp", n, sms, GRU_WARPS)[0] == min(wpb, GRU_WARPS)
    return n


def observe(env):
    nw = env.world.native
    return [o.clone() for o in nw.observe(out=nw.new_outputs(), flags=env._flags()).obs]


def model_of(actor, nw):
    from multiagent_particle_envs_b200.environment import rmappo_actor_params
    params, tanh, fn, eps = rmappo_actor_params([actor] * nw.n_agents, nw.obs_dims, nw.act_dims)
    net = ((FEATURE_NORM if fn else 0) | (TANH if tanh else 0), eps)
    return RecurrentModel([t.to(torch.float32).cpu().numpy() for t in params], net)


def check_replay_and_numerics(tag, n, T, explore, tanh, fn):
    env_a, env_b = twins(tag, n)
    na, nb = env_a.world.native, env_b.world.native
    A, act_dims, segs = env_a.n, list(na.act_dims), segments_of(env_a)
    actor = make_rmappo_actor(na.obs_dims[0], act_dims[0], tanh, fn)
    model = model_of(actor, na)
    seed = 0x1234_5678_9ABC if explore else None
    obs_b = observe(env_b)
    obs_r, rew_r, done_r, _, ex = env_a.rollout_policy([actor] * A, T, explore_seed=seed, action_mode="categorical",
                                                       **RECORDS)
    idx, logp, rew_steps, obs_rec = ex["actions"], ex["log_probs"], ex["rewards"], ex["observations"]
    hrec, hfin = ex["rnn_states"], ex["final_rnn_states"]
    assert tuple(hrec.shape) == (T, A, n, H) and tuple(hfin.shape) == (A, n, H) and hfin.dtype == torch.float32
    assert not bool(hrec[0].any())                                       # rnn_states=None: h starts at zero
    rew_sum = torch.zeros(A, n, device="cuda")
    flips = gaps = 0
    lmax = tight_max = loose_max = 0.0
    tight_in = total = 0
    stride = 2 if max(act_dims) <= 8 else 4
    for t in range(T):
        for i in range(A):
            assert torch.equal(obs_rec[i][t], obs_b[i]), (t, i)
            o = obs_b[i].cpu().numpy()
            h = hrec[t, i].cpu().numpy().astype(np.float64)
            hk = (hrec[t + 1, i] if t + 1 < T else hfin[i]).cpu().numpy().astype(np.float64)
            hm = model.gru(model.base(o), h)
            d = np.abs(hk - hm)
            tight, loose = model.h_bound(o, h, False), model.h_bound(o, h, True)
            assert (d <= loose).all(), (t, i, float((d - loose).max()))
            tight_in += int((d <= tight).sum())
            total += d.size
            tight_max, loose_max = max(tight_max, float(tight.max())), max(loose_max, float(loose.max()))
            g = gumbel_noise(seed, 0, np.arange(n), t, i, A, n_logits=act_dims[i], stride=stride) if explore else 0.0
            k = idx[i][t].cpu().numpy()
            lp = logp[t, i].cpu().numpy().astype(np.float64)
            f, gp = explain_head_mismatches(k, lp, hk, model, segs[i], noise=g)
            flips, gaps = flips + f, gaps + gp
            z64, _ = module_step(actor, o, h)
            err = np.abs(lp - log_softmax_at(z64, k, segs[i]))
            lmax = max(lmax, float(err.max()))
            dz = np.abs(model.logits(hk) - z64)          # the kernel's logits follow from its own h'
            bound = sum(2.0 * dz[:, a:b].max(-1) for a, b in bounds(segs[i])) + LOGP_FLIP_SLACK
            assert (err <= bound).all(), (t, i, float((err - bound).max()))
        obs_b, rew_s, _, _ = env_b.step([one_hot_torch(k[t], s) for k, s in zip(idx, segs)])
        rew_sum += torch.stack(list(rew_s))
        assert torch.equal(rew_steps[t], torch.stack(list(rew_s))), t
    torch.cuda.synchronize()
    assert torch.equal(na.agent_pv, nb.agent_pv)
    assert torch.equal(na.comm, nb.comm)
    for x, y in zip(obs_r, obs_b):
        assert torch.equal(x, y)
    assert torch.equal(torch.stack(list(rew_r)), rew_sum)
    assert not any(bool(x.any()) for x in done_r)
    assert env_a.explore_epoch == (1 if explore else 0)
    share = tight_in / total
    print("\nrmappo %s tanh=%s feature_norm=%s n=%d explore=%s: h' within the flip-free bound (max %.2e) for %.4f of "
          "entries, all within the bound with flips (max %.2e); %d of %d rows explained by TF32 flips of LN(h'), %d by "
          "the Gumbel gap; log-probabilities within %.3e of the unfolded float64 modules"
          % (tag, tanh, fn, n, explore, tight_max, share, loose_max, flips, n * T * A, gaps, lmax))
    assert share >= TIGHT_SHARE, share


@pytest.mark.parametrize("tag", GRU_PROGRAMS)
@pytest.mark.parametrize("tanh", [False, True])
@pytest.mark.parametrize("explore", [True, False])
def test_rmappo_replay_and_numerics(tag, tanh, explore):
    """a ragged multi-warp launch: 5-warp blocks with a partial last block and a partial last warp; the input
    LayerNorm is on for (ReLU, exploring) and (tanh, greedy)"""
    check_replay_and_numerics(tag, size(5), 3, explore, tanh, fn=(explore != tanh))


@pytest.mark.parametrize("tag,tanh,explore", [("simple_spread_n3", False, True), ("simple_reference", True, False)])
def test_rmappo_replay_at_the_block_cap(tag, tanh, explore):
    """65 536 worlds plus a ragged tail in blocks at the kernel's cap"""
    check_replay_and_numerics(tag, size(GRU_WARPS, base=65536), 2, explore, tanh, fn=True)


KEYS = ("rewards", "log_probs", "rnn_states")
LIST_KEYS = ("actions", "observations")


def test_hidden_state_carries_over_between_calls():
    """rollout_policy(T1 + T2) == rollout_policy(T1), then rollout_policy(T2, rnn_states=final_rnn_states), bit for
    bit; rnn_states=None == zeros"""
    tag, T1, T2 = "simple_spread_n3", 3, 4
    n = size(3)
    env_a, env_b = twins(tag, n)
    actor = make_rmappo_actor(18, 5, True, True)
    pols = [actor] * 3
    kw = dict(action_mode="categorical", **RECORDS)
    ra = env_a.rollout_policy(pols, T1 + T2, **kw)
    rb1 = env_b.rollout_policy(pols, T1, **kw)
    h1 = rb1[4]["final_rnn_states"].clone()
    rb2 = env_b.rollout_policy(pols, T2, rnn_states=h1, **kw)
    torch.cuda.synchronize()
    assert torch.equal(h1, rb1[4]["final_rnn_states"])                  # the input is never written
    for key in KEYS:
        assert torch.equal(ra[4][key], torch.cat([rb1[4][key], rb2[4][key]])), key
    for key in LIST_KEYS:
        for x, y1, y2 in zip(ra[4][key], rb1[4][key], rb2[4][key]):
            assert torch.equal(x, torch.cat([y1, y2])), key
    assert torch.equal(ra[4]["final_rnn_states"], rb2[4]["final_rnn_states"])
    assert torch.equal(rb2[4]["rnn_states"][0], h1)
    for x, y in zip(ra[0], rb2[0]):
        assert torch.equal(x, y)
    for x, y in zip(state(env_a), state(env_b)):
        assert torch.equal(x, y)
    env_c, env_d = twins(tag, n)
    rc = env_c.rollout_policy(pols, T1, **kw)
    rd = env_d.rollout_policy(pols, T1, rnn_states=torch.zeros(3, n, H, device="cuda"), **kw)
    torch.cuda.synchronize()
    for key in KEYS + ("final_rnn_states",):
        assert torch.equal(rc[4][key], rd[4][key]), key
    for x, y in zip(state(env_c), state(env_d)):
        assert torch.equal(x, y)


def rmappo_loop(env, pols, E, L, seed):
    parts = {k: [] for k in KEYS + LIST_KEYS}
    finals, rets = [], []
    for _ in range(E):
        obs_e, rew_e, _, _, ex = env.rollout_policy(pols, L, explore_seed=seed, action_mode="categorical", **RECORDS)
        for k in parts:
            parts[k].append(ex[k])
        finals.append(obs_e)
        rets.append(rew_e)
        h_final = ex["final_rnn_states"]
        obs = env.reset()
    A = env.n
    out = dict(obs=obs, final=[torch.stack([f[i] for f in finals]) for i in range(A)],
               returns=[torch.stack([r[i] for r in rets]) for i in range(A)], final_rnn_states=h_final)
    out.update({k: torch.cat(parts[k]) for k in KEYS})
    out.update({k: [torch.cat([a[i] for a in parts[k]]) for i in range(A)] for k in LIST_KEYS})
    return out


@pytest.mark.parametrize("tag", GRU_PROGRAMS)
@pytest.mark.parametrize("E,L,explore,tanh,fn", [(3, 4, True, True, True), (2, 3, False, False, False)])
def test_rmappo_episodes_equal_the_loop(tag, E, L, explore, tanh, fn):
    n = size(5)
    env_a, env_b = twins(tag, n)
    nw = env_a.world.native
    pols = [make_rmappo_actor(nw.obs_dims[0], nw.act_dims[0], tanh, fn)] * env_a.n
    seed = 21 if explore else None
    epoch = nw.epoch
    obs, ret, done, _, ex = env_a.rollout_policy(pols, E * L, episode_length=L, explore_seed=seed,
                                                 action_mode="categorical", **RECORDS)
    ref = rmappo_loop(env_b, pols, E, L, seed)
    torch.cuda.synchronize()
    for e in range(E):
        assert not bool(ex["rnn_states"][e * L].any()), e                # every episode starts from h = 0
    for key in KEYS + ("final_rnn_states",):
        assert torch.equal(ex[key], ref[key]), key
    for key in LIST_KEYS:
        for i in range(env_a.n):
            assert torch.equal(ex[key][i], ref[key][i]), (key, i)
    for i in range(env_a.n):
        assert torch.equal(ex["final_observations"][i], ref["final"][i]), ("final observations", i)
        assert torch.equal(ret[i], ref["returns"][i]), ("returns", i)
        assert torch.equal(obs[i], ref["obs"][i]), ("post-reset observations", i)
        assert not bool(done[i].any())
    for x, y in zip(state(env_a), state(env_b)):
        assert torch.equal(x, y)
    assert nw.epoch == env_b.world.native.epoch == epoch + E
    assert env_a.explore_epoch == env_b.explore_epoch == (E if explore else 0)


def test_refusals_leave_state_and_epochs_unchanged():
    from multiagent_particle_envs_b200._lib import MpeError
    env = make_product_env("simple_spread_n3", num_envs=64, seed=9)
    env.reset()
    nw = env.world.native
    actor = make_rmappo_actor(18, 5, False, True)
    before, epoch = state(env), nw.epoch

    def unchanged(e, b, ep):
        torch.cuda.synchronize()
        for x, y in zip(state(e), b):
            assert torch.equal(x, y)
        assert e.world.native.epoch == ep and e.explore_epoch == 0

    cat = dict(action_mode="categorical", explore_seed=1, record_log_probs=True)
    with pytest.raises(NotImplementedError, match="categorical"):
        env.rollout_policy([actor] * 3, 4, explore_seed=1)
    unchanged(env, before, epoch)
    with pytest.raises(NotImplementedError, match="shared"):          # equal values, distinct tuples
        env.rollout_policy([actor, tuple(list(actor)), tuple(list(actor))], 4, **cat)
    unchanged(env, before, epoch)
    bad = (actor[0], torch.nn.GRU(64, 64, num_layers=2).cuda(), actor[2], actor[3])
    with pytest.raises(ValueError, match="num_layers=1"):
        env.rollout_policy([bad] * 3, 4, **cat)
    unchanged(env, before, epoch)
    for h0 in (torch.zeros(3, 64, 32, device="cuda"), torch.zeros(3, 64, H, device="cuda", dtype=torch.float64),
               torch.zeros(3, 64, H), torch.zeros(2, 64, H, device="cuda")):
        with pytest.raises(ValueError, match="rnn_states"):
            env.rollout_policy([actor] * 3, 4, rnn_states=h0, **cat)
        unchanged(env, before, epoch)
    with pytest.raises(ValueError, match="episode_length"):
        env.rollout_policy([actor] * 3, 4, episode_length=2, rnn_states=torch.zeros(3, 64, H, device="cuda"), **cat)
    unchanged(env, before, epoch)
    tag = make_product_env("simple_tag", num_envs=64, seed=9)          # a program without the kernel
    tag.reset()
    tnw = tag.world.native
    tbefore, tepoch = state(tag), tnw.epoch
    shared = make_rmappo_actor(tnw.obs_dims[0], tnw.act_dims[0], True, False)
    for kw in ({}, {"episode_length": 2}):
        with pytest.raises(MpeError, match="no compiled"):
            tag.rollout_policy([shared] * tag.n, 4, **cat, **kw)
        unchanged(tag, tbefore, tepoch)
