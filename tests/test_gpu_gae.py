"""env.compute_gae (mpe_gae) on the GPU: returns and raw advantages bit-identical to the float32 mirror (seeded inputs at
a ragged size, one episode and the episode form; the real outputs of rollout_policy with MAPPO's critic and with
rMAPPO's recurrent critic), returns within the mirror's derived float32 bound of MAPPO's float64 loop, the normalised
advantages bit-identical to the mirror given the reported (mean, std) and (mean, std) against float64 NumPy, two
calls bit-identical, a CUDA-graph replay equal to the eager call, inputs untouched, and a buffer of more than 2^31
entries."""
import numpy as np
import pytest

from critic_helpers import make_critic
from gae_helpers import gae_mirror, mappo_returns, normalize_mirror, seeded_inputs
from helpers import make_product_env
from mappo_helpers import make_mappo_actors
from rcritic_helpers import make_rcritic
from rmappo_helpers import make_rmappo_actor

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

GAMMA, LAM = 0.99, 0.95


def cuda(*arrays):
    return [None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]


def check_stats(stats, adv):
    """(mean, std) within 1e-9 relative of float64 NumPy over the raw advantages (the mean relative to |mean| + std:
    its own size may be anything)"""
    a = adv.astype(np.float64)
    mean, std = float(stats[0]), float(stats[1])
    assert abs(mean - a.mean()) <= 1e-9 * (abs(a.mean()) + a.std())
    assert abs(std - a.std()) <= 1e-9 * a.std()


def check_normalized(norm, raw, stats):
    assert np.array_equal(norm, normalize_mirror(raw, float(stats[0]), float(stats[1])))


@pytest.mark.parametrize("value_norm", [None, "shared", "per_agent"])
@pytest.mark.parametrize("bootstrap", [True, False])
@pytest.mark.parametrize("T,L", [(25, None), (200, 25)])
def test_seeded_inputs_match_the_mirror(T, L, bootstrap, value_norm):
    """65 553 worlds of simple_spread N=3 (a ragged last block): returns and raw advantages bit for bit, returns within
    the derived bound of MAPPO's float64 loop, then the normalised call against the mirror and float64 NumPy"""
    N = 65553
    env = make_product_env("simple_spread_n3", num_envs=N)
    n, E = env.n, 1 if L is None else T // L
    rew, val, final, vn = seeded_inputs(T, n, N, E, seed=T + bootstrap, per_agent_norm=value_norm == "per_agent")
    vn = None if value_norm is None else vn
    final_in = final[0] if L is None else final
    r_d, v_d, f_d, vn_d = cuda(rew, val, final_in if bootstrap else None, vn)
    ret, adv, stats = env.compute_gae(r_d, v_d, f_d, gamma=GAMMA, gae_lambda=LAM, episode_length=L,
                                      bootstrap=bootstrap, value_norm=vn_d)
    assert stats is None and ret.shape == adv.shape == (T, n, N) and ret.dtype == torch.float32
    want_ret, want_adv, bound = gae_mirror(rew, val, final, GAMMA, LAM, L, bootstrap, vn)
    got_ret, got_adv = ret.cpu().numpy(), adv.cpu().numpy()
    assert np.array_equal(got_ret, want_ret) and np.array_equal(got_adv, want_adv)
    exact = mappo_returns(rew, val, final, GAMMA, LAM, L, bootstrap, vn)
    assert (np.abs(got_ret.astype(np.float64) - exact) <= bound + 1e-12 * (1 + np.abs(exact))).all()
    ret2, adv2, stats2 = env.compute_gae(r_d, v_d, f_d, gamma=GAMMA, gae_lambda=LAM, episode_length=L,
                                         bootstrap=bootstrap, value_norm=vn_d, normalize_advantages=True)
    assert stats2.dtype == torch.float64 and stats2.shape == (2,)
    assert torch.equal(ret2, ret)
    s = stats2.cpu().numpy()
    check_stats(s, got_adv)
    check_normalized(adv2.cpu().numpy(), got_adv, s)
    # the inputs are read only
    for d, h in ((r_d, rew), (v_d, val), (f_d, final_in), (vn_d, vn)):
        if d is not None:
            assert np.array_equal(d.cpu().numpy(), h)


def test_two_calls_are_identical_and_a_graph_replay_equals_the_eager_call():
    """the fixed-order reduction gives the same bits twice; a captured call replays on new inputs as the eager call"""
    N, T, L = 4099, 50, 25
    env = make_product_env("simple_spread_n3", num_envs=N)
    rew, val, final, vn = seeded_inputs(T, env.n, N, 2, seed=5, per_agent_norm=True)
    r_d, v_d, f_d, vn_d = cuda(rew, val, final, vn)
    kw = dict(episode_length=L, value_norm=vn_d, normalize_advantages=True)
    a = env.compute_gae(r_d, v_d, f_d, **kw)
    b = env.compute_gae(r_d, v_d, f_d, **kw)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        env.compute_gae(r_d, v_d, f_d, **kw)   # warm-up on the capturing stream
        with torch.cuda.graph(g, stream=side):
            cap = env.compute_gae(r_d, v_d, f_d, **kw)
    torch.cuda.current_stream().wait_stream(side)
    rew2, val2, final2, vn2 = seeded_inputs(T, env.n, N, 2, seed=6, per_agent_norm=True)
    for d, h in zip((r_d, v_d, f_d, vn_d), (rew2, val2, final2, vn2)):
        d.copy_(torch.from_numpy(h))
    g.replay()
    eager = env.compute_gae(r_d, v_d, f_d, **kw)
    torch.cuda.synchronize()
    for x, y in zip(cap, eager):
        assert torch.equal(x, y)
    want_ret, want_adv, _ = gae_mirror(rew2, val2, final2, GAMMA, LAM, L, True, vn2)
    assert np.array_equal(cap[0].cpu().numpy(), want_ret)
    check_normalized(cap[1].cpu().numpy(), want_adv, cap[2].cpu().numpy())


def check_rollout(env, ex, L=None, vn=None):
    """compute_gae over a rollout's extras (rewards, values, final_values) against the mirror, with and without a
    per-agent ValueNorm"""
    rew, val, fin = (ex[k].cpu().numpy() for k in ("rewards", "values", "final_values"))
    for value_norm in (None, vn):
        vn_d = None if value_norm is None else torch.from_numpy(value_norm).cuda()
        ret, adv, _ = env.compute_gae(ex["rewards"], ex["values"], ex["final_values"], gamma=GAMMA, gae_lambda=LAM,
                                      episode_length=L, value_norm=vn_d)
        want_ret, want_adv, _ = gae_mirror(rew, val, fin, GAMMA, LAM, L, True, value_norm)
        assert np.array_equal(ret.cpu().numpy(), want_ret) and np.array_equal(adv.cpu().numpy(), want_adv)


def per_agent_norm(n):
    return np.stack([np.linspace(-3.0, -1.0, n), np.linspace(0.5, 2.0, n)], 1).astype(np.float32)


@pytest.mark.parametrize("tag,per_agent", [("simple_spread_n3", False), ("simple_tag", False),
                                           ("simple_speaker_listener", True)])
def test_on_the_mappo_critics_rollout(tag, per_agent):
    """rollout_policy with MAPPO's critic (shared, or one per agent): its rewards, values and final values"""
    N = 1000
    env = make_product_env(tag, num_envs=N, seed=3)
    env.reset()
    nw = env.world.native
    actors = make_mappo_actors(nw.obs_dims, nw.act_dims, False, True)
    critic = [make_critic(nw.obs_dims, False, True, seed=11 + i) for i in range(env.n)] if per_agent else \
        make_critic(nw.obs_dims, False, True)
    ex = env.rollout_policy(actors, 25, explore_seed=1, action_mode="categorical", per_step_rewards=True,
                            critic=critic)[4]
    check_rollout(env, ex, vn=per_agent_norm(env.n))


def test_on_the_rmappo_critics_episodes():
    """rollout_policy with rMAPPO's recurrent critic in the episode form: [E, n, N] final values"""
    N, E, L = 1000, 4, 25
    env = make_product_env("simple_spread_n3", num_envs=N, seed=3)
    env.reset()
    nw = env.world.native
    actor = make_rmappo_actor(nw.obs_dims[0], nw.act_dims[0], False, True)
    critic = make_rcritic(nw.obs_dims, False, True)
    ex = env.rollout_policy([actor] * env.n, E * L, episode_length=L, explore_seed=2, action_mode="categorical",
                            per_step_rewards=True, critic=critic)[4]
    assert tuple(ex["final_values"].shape) == (E, env.n, N)
    check_rollout(env, ex, L=L, vn=per_agent_norm(env.n))


def test_refuses_tensors_on_the_host():
    env = make_product_env("simple_spread_n3", num_envs=64)
    env.reset()
    x = torch.zeros(4, 3, 64)
    with pytest.raises(ValueError, match="CUDA tensor"):
        env.compute_gae(x, x, x[0])
    with pytest.raises(ValueError, match="value_norm must be a CUDA tensor"):
        y = x.cuda()
        env.compute_gae(y, y, y[0], value_norm=torch.zeros(2))


def test_more_than_2_31_entries():
    """simple_spread N=3 at 65 536 worlds and T = 11 000: 2 162 688 000 entries, 8.7 GB per [T, n, N] array (about
    35 GB for rewards, values, returns and advantages).  Every step of the first and last 32 worlds of every agent
    against the mirror (the entries past 2^31 are the last steps), and (mean, std) against float64 sums of the whole
    buffer"""
    N, T = 65536, 11000
    env = make_product_env("simple_spread_n3", num_envs=N)
    n = env.n
    assert T * n * N > 2 ** 31
    g = torch.Generator(device="cuda").manual_seed(1)
    rew = torch.randn(T, n, N, device="cuda", generator=g).mul_(0.5).sub_(1.0)
    val = torch.randn(T, n, N, device="cuda", generator=g)
    fin = torch.randn(n, N, device="cuda", generator=g)
    vn = torch.tensor([-10.0, 4.0], device="cuda")
    cols = np.r_[0:32, N - 32:N]

    def host(t):
        return t[..., cols].cpu().numpy()

    r_h, v_h, f_h = host(rew), host(val), host(fin)
    ret, adv, _ = env.compute_gae(rew, val, fin, value_norm=vn)
    want_ret, want_adv, _ = gae_mirror(r_h, v_h, f_h, 0.99, 0.95, None, True, vn.cpu().numpy())
    raw = host(adv)
    assert np.array_equal(host(ret), want_ret) and np.array_equal(raw, want_adv)
    s = s2 = 0.0
    for chunk in adv.split(500):
        c = chunk.double()
        s += float(c.sum())
        s2 += float(c.pow_(2).sum())
    m = float(T * n * N)
    mean, std = s / m, np.sqrt(s2 / m - (s / m) ** 2)
    del ret, adv
    torch.cuda.empty_cache()
    _, norm, stats = env.compute_gae(rew, val, fin, value_norm=vn, normalize_advantages=True)
    st = stats.cpu().numpy()
    assert abs(st[0] - mean) <= 1e-9 * (abs(mean) + std) and abs(st[1] - std) <= 1e-9 * std
    check_normalized(host(norm), raw, st)


def test_entry_point_refuses_each_bad_argument_on_a_device():
    """mpe_gae on a bound handle: every check after the device's (episode length, gamma and lambda, flags, pointers,
    workspace size and alignment) returns MPE_ERR_BAD_ARG and writes nothing; a workspace that is 8 but not 16-byte
    aligned is accepted and gives the aligned call's results"""
    from multiagent_particle_envs_b200 import _lib
    lib = _lib.load()
    BAD_ARG = -1
    N, T = 300, 8
    env = make_product_env("simple_spread_n3", num_envs=N)
    env.reset()
    h = env.world.native.handle
    rew, val, fin, vn = cuda(*seeded_inputs(T, env.n, N, 1, seed=2)[:3], np.array([-1.0, 2.0], np.float32))
    ret = torch.full((T, env.n, N), 7.0, device="cuda")
    adv = torch.full((T, env.n, N), 7.0, device="cuda")
    wsb = lib.mpe_gae_workspace_bytes(h)
    ws = torch.zeros(wsb // 8 + 2, dtype=torch.float64, device="cuda")   # 256-byte aligned base
    base = dict(r=rew.data_ptr(), v=val.data_ptr(), f=fin.data_ptr(), steps=T, L=0, gamma=GAMMA, lam=LAM, flags=3,
                vn=vn.data_ptr(), ret=ret.data_ptr(), adv=adv.data_ptr(), ws=ws.data_ptr(), wsb=wsb)

    def call(**kw):
        d = dict(base, **kw)
        return lib.mpe_gae(h, d["r"], d["v"], d["f"], d["steps"], d["L"], d["gamma"], d["lam"], d["flags"], d["vn"],
                           d["ret"], d["adv"], d["ws"], d["wsb"], None)

    probes = [dict(steps=0), dict(L=3), dict(L=-1), dict(gamma=1.5), dict(gamma=float("inf")), dict(lam=float("nan")),
              dict(lam=-0.5), dict(flags=8), dict(r=None), dict(r=base["r"] + 2), dict(v=None), dict(ret=None),
              dict(adv=base["adv"] + 1), dict(f=None), dict(f=base["f"] + 2), dict(vn=base["vn"] + 2),
              dict(flags=7, vn=None), dict(ws=None), dict(ws=base["ws"] + 4), dict(wsb=wsb - 1)]
    assert [call(**kw) for kw in probes] == [BAD_ARG] * len(probes)
    torch.cuda.synchronize()
    assert bool((ret == 7.0).all()) and bool((adv == 7.0).all())
    assert call(flags=2, f=None) == 0 and call(flags=0, f=None, ws=None, wsb=0) == 0   # no bootstrap / no workspace
    assert call() == 0
    torch.cuda.synchronize()
    ret_a, adv_a, stats_a = ret.clone(), adv.clone(), ws[:2].clone()
    ret.fill_(7.0)
    adv.fill_(7.0)
    assert call(ws=base["ws"] + 8) == 0   # 8 mod 16: the partials are read and written as single doubles
    torch.cuda.synchronize()
    assert torch.equal(ret, ret_a) and torch.equal(adv, adv_a) and torch.equal(ws[1:3], stats_a)
