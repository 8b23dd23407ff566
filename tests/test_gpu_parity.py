"""Parity of the sm_90a kernels (through the C ABI / the reference-shaped Python API) against
(a) the committed golden fixtures produced by the real reference, and (b) the CPU oracle on seeded
synthetic worlds.  Tolerance for fp32 vs the fp64 reference: rtol 1e-5, atol 1e-6 per step
(BASELINE.json north_star); collision counts / done masks bit-exact vs the fp32 oracle evaluated
on the kernels' own stored state.  Run on an H100: pytest -m gpu."""
import numpy as np
import pytest

from helpers import (CONFIGS, PROGRAM_TAGS, STEP_DENSE_TAGS, VARIANTS, VELOCITY_TERM_ULPS, explain_flag_mismatches,
                     load_golden, make_product_env, random_actions, random_goals, random_states, scenario_of, split_cols,
                     velocity_term_scale)

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

RTOL, ATOL = 1e-5, 1e-6
TAGS = list(CONFIGS)


def inject(nw, pv, lm, comm, goal=None):
    """oracle layout [n,A,4] / [n,L,2] / [n,A,C] / [n,G] -> the SoA device tensors"""
    dev = nw.device
    if goal is not None and nw.n_goals:
        nw.goal.copy_(torch.as_tensor(np.ascontiguousarray(goal), dtype=torch.int32, device=dev).t())
    nw.agent_pv.copy_(torch.as_tensor(pv, dtype=torch.float32, device=dev).permute(1, 0, 2))
    if nw.n_landmarks:
        nw.lm_p.copy_(torch.as_tensor(lm, dtype=torch.float32, device=dev).permute(1, 0, 2))
    C = nw.dim_c
    for i in range(nw.n_agents):
        s = nw.speaker_slot(i)
        if s >= 0 and C:
            nw.comm[s * C:(s + 1) * C].copy_(torch.as_tensor(comm[:, i, :], dtype=torch.float32, device=dev).t())


def extract(nw):
    pv = nw.agent_pv.permute(1, 0, 2).cpu().numpy()
    C = nw.dim_c
    comm = np.zeros((nw.n_env, nw.n_agents, C), np.float32)
    for i in range(nw.n_agents):
        s = nw.speaker_slot(i)
        if s >= 0 and C:
            comm[:, i, :] = nw.comm[s * C:(s + 1) * C].t().cpu().numpy()
    return pv, comm


def gpu_step(env, act, flags_expected=None):
    """act: [n, sum_act] -> CUDA step -> numpy (obs [n,sum_obs], rew [n,A], done [n,A], info [n,A,I])"""
    nw = env.world.native
    if env.discrete_action_input:       # one integer column per sub-action, int32 straight into the kernel
        subs = [len(s) for s in env._sub_sizes]
        acts = [torch.as_tensor(np.ascontiguousarray(a), device=nw.device).to(torch.int32) for a in split_cols(act, subs)]
    else:
        acts = [torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float32, device=nw.device)
                for a in split_cols(act, nw.act_dims)]
    obs_n, rew_n, done_n, info_n = env.step(acts)
    torch.cuda.synchronize()
    obs = np.concatenate([o.cpu().numpy() for o in obs_n], axis=1)
    rew = torch.stack(rew_n, 1).cpu().numpy()
    done = torch.stack(done_n, 1).cpu().numpy().astype(np.uint8)
    out = env._last_out
    info = out.info.permute(2, 0, 1).cpu().numpy() if out.info is not None else np.zeros((nw.n_env, nw.n_agents, 0))
    return obs, rew, done, info


# reference worlds with other entity counts
GOLDEN_VARIANTS = ["simple_tag_1v1", "simple_tag_4v2", "simple_tag_6v2", "simple_tag_2v1", "simple_spread_n2",
                   "simple_spread_n4", "simple_spread_n5", "simple_adversary_n4"]


@pytest.mark.parametrize("tag", TAGS + ["simple_tag_force_discrete", "simple_tag_discrete_input"] + GOLDEN_VARIANTS)
def test_golden_fixtures_single_step(tag):
    """every recorded reference step (>= 1536 per scenario, 256 worlds, half of them in contact equilibrium), state
    re-injected each step (BASELINE.md 4.4)"""
    g = load_golden(tag)
    base = tag if tag in VARIANTS else ("simple_tag" if tag.startswith("simple_tag") else tag)
    W, T = g["act"].shape[:2]
    env = make_product_env(base, num_envs=W)
    env.force_discrete_action = bool(int(g["force_discrete"]))
    env.discrete_action_input = bool(int(g["discrete_input"]))
    env.reset()
    nw = env.world.native
    flipped = 0
    for t in range(T):
        inject(nw, g["pv0"] if t == 0 else g["pv"][:, t - 1], g["lm"], g["comm0"] if t == 0 else g["comm"][:, t - 1],
               g.get("goal"))
        obs, rew, done, info = gpu_step(env, g["act"][:, t])
        pv, comm = extract(nw)
        np.testing.assert_allclose(pv, g["pv"][:, t], rtol=RTOL, atol=ATOL)
        np.testing.assert_allclose(comm, g["comm"][:, t], rtol=1e-7, atol=0)
        np.testing.assert_allclose(obs, g["obs"][:, t], rtol=RTOL, atol=ATOL)
        assert np.array_equal(done, g["done"][:, t])
        # a contact flag evaluated in fp32 may differ from fp64 when the distance is within rounding of its threshold:
        # every reward / info mismatch must be exactly that (integer multiple of the contact quantum AND a pair within
        # 2e-6 of a threshold in the fp64 golden state) -- anything else fails
        flipped += explain_flag_mismatches(tag, rew, g["rew"][:, t], info if info.shape[2] else None,
                                           g["info"][:, t] if info.shape[2] else None, g["pv"][:, t], g["lm"],
                                           g["prop_agent_size"], g["prop_landmark_size"])
    assert flipped <= max(2, W * T // 200), flipped


@pytest.mark.parametrize("tag", TAGS)
def test_golden_fixtures_free_running(tag):
    """25-step trajectories without re-injection stay close (loose: contacts amplify rounding)"""
    g = load_golden(tag)
    W, T = g["act"].shape[:2]
    env = make_product_env(tag, num_envs=W)
    env.reset()
    nw = env.world.native
    inject(nw, g["pv0"], g["lm"], g["comm0"], g.get("goal"))
    for t in range(T):
        obs, rew, done, info = gpu_step(env, g["act"][:, t])
    pv, _ = extract(nw)
    err = np.abs(pv - g["pv"][:, T - 1])
    assert np.median(err) < 1e-5 and (err < 1e-3).mean() > 0.97


def close_per_element(got, want, slack=0.0):
    """rtol 1e-5 / atol 1e-6 per element, or within `slack` (per element) where the value is ill-conditioned"""
    err = np.abs(got - want)
    bad = err > np.maximum(ATOL + RTOL * np.abs(want), slack)
    assert not bad.any(), ("%d elements beyond rtol %g / atol %g: first %s, |difference| %s" % (
        int(bad.sum()), RTOL, ATOL, np.argwhere(bad)[:4].tolist(), err[bad][:4]))


@pytest.mark.parametrize("tag,n", [("simple", 4096), ("simple_spread_n3", 8192), ("simple_spread_n6", 4096),
                                   ("simple_tag", 8192), ("simple_world_comm", 4096), ("simple_adversary", 4096),
                                   ("simple_push", 4096), ("simple_speaker_listener", 4096), ("simple_reference", 4096),
                                   ("simple_crypto", 4096), ("simple_tag_1v1", 2048), ("simple_tag_2v1", 2048),
                                   ("simple_tag_4v2", 2048), ("simple_tag_6v2", 2048), ("simple_adversary_n4", 2048),
                                   # production sizes (BASELINE.json) and launch shapes of the fused step, see
                                   # helpers.launch_shape "step": (hot kernel, warps per block) -- resolved on the device
                                   ("simple_spread_n3", 65536), ("simple_tag", 262144), ("simple_spread_n6", 131072),
                                   ("simple_world_comm", 32768), ("simple_tag", "dense_4warp_ragged")]
                         # every program: 1-warp blocks of the HOT kernel and the general kernel's ragged tail
                         + [(tag, "1warp_ragged") for tag in PROGRAM_TAGS]
                         # the 80-register builds in 2- and 4-warp blocks, partial last block, ragged tail
                         + [(tag, r) for tag in STEP_DENSE_TAGS for r in ("dense_2warp_ragged", "dense_4warp_ragged")
                            if (tag, r) != ("simple_tag", "dense_4warp_ragged")])
def test_seeded_worlds_vs_oracle(tag, n):
    from oracle import Oracle
    from multiagent_particle_envs_b200 import _lib
    from helpers import device_sms, launch_shape, regime_size, step_uses_dense
    sms = device_sms()
    if n == "1warp_ragged":           # 1-warp blocks of the 128-register HOT kernel + the general kernel's 17-world tail
        n = regime_size("step", sms, 1, base=2048)
        assert not step_uses_dense(tag, n, sms) and launch_shape("step", n, sms)[0] == 1 and n % 32 == 17
    elif n in ("dense_2warp_ragged", "dense_4warp_ragged"):   # the 80-register kernel + the general kernel's tail
        wpb = int(n[6])
        n = regime_size("step", sms, wpb)
        assert step_uses_dense(tag, n, sms) and launch_shape("step", n, sms)[:3:2] == (wpb, True) and n % 32
    elif n == 262144:                 # the BASELINE tag size: 80-register kernel, 2-warp blocks on 132 SMs (4 on 114)
        assert step_uses_dense(tag, n, sms) and launch_shape("step", n, sms)[0] == 2
    elif n == 131072:                 # the BASELINE spread N=6 size: 2-warp blocks (on 64 SMs or more)
        assert not step_uses_dense(tag, n, sms) and launch_shape("step", n, sms)[0] == 2
    env = make_product_env(tag, num_envs=n)
    env.reset()
    nw = env.world.native
    desc = env.world.descriptor()
    o64, o32 = Oracle(desc, "f64"), Oracle(desc, "f32")
    flags = _lib.FLAG_SHARED_REWARD if env.shared_reward else 0
    rng = np.random.RandomState(1234)
    pv0, lm, comm0 = random_states(desc, n, rng)
    pv0, lm, comm0 = pv0.astype(np.float32), lm.astype(np.float32), comm0.astype(np.float32)
    movable = [bool(desc.agent_movable[i]) for i in range(desc.n_agents)]
    act = random_actions(nw.act_dims, n, rng, movable=movable).astype(np.float32)
    goal = random_goals(nw.n_goals, desc.n_landmarks, n, rng) if nw.n_goals else None
    inject(nw, pv0, lm, comm0, goal)
    obs, rew, done, info = gpu_step(env, act)
    pv, comm = extract(nw)
    # (1) against the reference arithmetic (fp64) on identical fp32 inputs
    rpv, rcomm, robs, rrew, rdone, rinfo = o64.step(pv0, lm, comm0, act, flags, goal=goal)
    # a velocity that is the small difference of large contact forces (squeezed worlds) may differ by a few fp32 ulps of
    # those forces (seen: spread N=6 at 131 072 worlds, 1.19e-6 on a velocity of -0.0123 whose terms sum to 9.96 in
    # magnitude -- 2 ulps of them); the same slack applies to the observation entries that copy the velocity
    slack = VELOCITY_TERM_ULPS * 2.0 ** -24 * velocity_term_scale(desc, pv0, lm, act, nw.act_dims)
    pv_slack = np.zeros_like(rpv)
    pv_slack[:, :, 2:4] = slack
    obs_slack = np.zeros_like(robs)
    if scenario_of(tag) in ("simple", "simple_spread", "simple_tag", "simple_world_comm"):   # obs = [own vel, ...]
        for i, o in enumerate(np.cumsum([0] + list(nw.obs_dims))[:-1]):
            obs_slack[:, o:o + 2] = slack[:, i]
    close_per_element(pv, rpv, pv_slack)
    np.testing.assert_allclose(comm, rcomm, rtol=1e-7, atol=0)
    close_per_element(obs, robs, obs_slack)
    assert np.array_equal(done, rdone)
    a_size = [desc.agent_size[i] for i in range(desc.n_agents)]
    l_size = [desc.landmark_size[l] for l in range(desc.n_landmarks)]
    flipped = explain_flag_mismatches(tag, rew, rrew, None, None, rpv, lm, a_size, l_size)   # every mismatch is a flipped flag
    assert flipped <= max(2, n // 200), flipped
    # (2) flags: the fp32 oracle evaluated on the kernel's OWN stored post-step state must give
    # bit-identical observations, contact counts and done masks (SURVEY.md 7.4.3)
    fobs, frew, fdone, finfo = o32.observe(pv, lm, comm, flags, goal=goal)
    assert np.array_equal(obs, fobs)
    assert np.array_equal(done, fdone)
    count_cols = [1, 3] if tag.startswith("simple_spread") else ([0] if tag.startswith(("simple_tag", "simple_world_comm")) else [])
    for c in count_cols:                                              # collisions / occupied landmarks
        assert np.array_equal(info[:, :, c], finfo[:, :, c])
    np.testing.assert_allclose(rew, frew, rtol=2e-6, atol=2e-6)       # only expf ulps may differ
    # some worlds really are in contact, otherwise the test proves little
    if any(desc.agent_collide[i] for i in range(desc.n_agents)) and desc.n_agents > 1:
        floor = 0.003 if tag == "simple_push" else 0.05            # two small agents rarely touch
        assert (np.abs(rpv[:, :, 2:4] - pv0[:, :, 2:4] * 0.75).max(axis=(1, 2)) > 1.0).mean() > floor


@pytest.mark.parametrize("tag", PROGRAM_TAGS)
def test_fused_step_equals_three_kernel_path(tag):
    """mpe_step == mpe_set_action -> mpe_world_step -> mpe_observe, bit for bit"""
    from multiagent_particle_envs_b200 import _lib
    n = 3000
    env_a = make_product_env(tag, num_envs=n)
    env_b = make_product_env(tag, num_envs=n)
    env_a.reset()
    env_b.reset()
    na, nb = env_a.world.native, env_b.world.native
    desc = env_a.world.descriptor()
    rng = np.random.RandomState(7)
    pv0, lm, comm0 = random_states(desc, n, rng)
    movable = [bool(desc.agent_movable[i]) for i in range(desc.n_agents)]
    act = random_actions(na.act_dims, n, rng, movable=movable).astype(np.float32)
    goal = random_goals(na.n_goals, desc.n_landmarks, n, rng) if na.n_goals else None
    inject(na, pv0, lm, comm0, goal)
    inject(nb, pv0, lm, comm0, goal)
    obs, rew, done, info = gpu_step(env_a, act)
    acts = [torch.as_tensor(np.ascontiguousarray(a), device=nb.device) for a in split_cols(act, nb.act_dims)]
    flags = _lib.FLAG_SHARED_REWARD if env_b.shared_reward else 0
    nb.set_action(_lib.ptr_array([t.data_ptr() for t in acts]), flags)
    env_b.world.step()                      # World.step(), core.py:117
    out = nb.observe(flags=flags)
    torch.cuda.synchronize()
    assert torch.equal(na.agent_pv, nb.agent_pv)
    assert torch.equal(na.comm, nb.comm)
    assert np.array_equal(obs, np.concatenate([o.cpu().numpy() for o in out.obs], 1))
    assert np.array_equal(rew, out.rew.t().cpu().numpy())


def test_scalar_api_matches_reference_known_answers():
    """BASELINE config 1: `simple`, batch 1, the reference's calling convention end to end"""
    import os
    from helpers import GOLDEN
    from make_env import make_env
    k = dict(np.load(os.path.join(GOLDEN, "kat.npz")))
    for name in ("simple", "simple_spread", "simple_tag", "simple_world_comm"):
        env = make_env(name)
        obs_n = env.reset()
        assert isinstance(obs_n, list) and obs_n[0].dtype == np.float64 and obs_n[0].ndim == 1
        world = env.world
        for i, ag in enumerate(world.agents):           # inject through the reference's own attributes
            ag.state.p_pos = k[name + "/pv0"][i, 0:2]
            ag.state.p_vel = k[name + "/pv0"][i, 2:4]
        for l, lmk in enumerate(world.landmarks):
            lmk.state.p_pos = k[name + "/lm"][l]
        acts = split_cols(k[name + "/act"], [5 + (4 if (name == "simple_world_comm" and i == 0) else 0)
                                             for i in range(env.n)])
        for _ in range(2):
            obs_n, rew_n, done_n, info_n = env.step([a.copy() for a in acts])
        assert len(obs_n) == env.n and all(o.dtype == np.float64 for o in obs_n)
        assert all(isinstance(d, bool) for d in done_n) and not any(done_n)
        assert set(info_n) == {"n"} and len(info_n["n"]) == env.n
        np.testing.assert_allclose(np.concatenate(obs_n), k[name + "/obs"], rtol=RTOL, atol=ATOL)
        np.testing.assert_allclose(np.array(rew_n), k[name + "/rew"], rtol=RTOL, atol=ATOL)
        np.testing.assert_allclose(world.agents[0].state.p_pos, k[name + "/pv"][0, 0:2], rtol=RTOL, atol=ATOL)
        np.testing.assert_allclose(world.agents[0].state.p_vel, k[name + "/pv"][0, 2:4], rtol=RTOL, atol=ATOL)


@pytest.mark.parametrize("n", [1, 31, 32, 33, 127, 129, 1000])
def test_ragged_batch_sizes(n):
    """partial warps / partial blocks take the scalar tile path; results equal the big-batch rows"""
    from oracle import Oracle
    from multiagent_particle_envs_b200 import _lib
    tag = "simple_tag"
    env = make_product_env(tag, num_envs=n)
    env.reset()
    nw = env.world.native
    desc = env.world.descriptor()
    rng = np.random.RandomState(n)
    pv0, lm, comm0 = random_states(desc, n, rng)
    act = random_actions(nw.act_dims, n, rng).astype(np.float32)
    inject(nw, pv0, lm, comm0)
    obs, rew, done, info = gpu_step(env, act)
    pv, _ = extract(nw)
    rpv, _, robs, rrew, rdone, _ = Oracle(desc, "f64").step(pv0.astype(np.float32), lm.astype(np.float32),
                                                             comm0, act, 0)
    np.testing.assert_allclose(pv, rpv, rtol=RTOL, atol=ATOL)
    np.testing.assert_allclose(obs, robs, rtol=RTOL, atol=ATOL)


def test_unaligned_action_views_are_handled():
    """non-contiguous / misaligned action tensors are normalised by the wrapper, not rejected"""
    n = 96
    env_a = make_product_env("simple_spread_n3", num_envs=n)
    env_b = make_product_env("simple_spread_n3", num_envs=n)
    env_a.reset()
    env_b.reset()
    env_b.world.native.agent_pv.copy_(env_a.world.native.agent_pv)
    env_b.world.native.lm_p.copy_(env_a.world.native.lm_p)
    big = torch.rand(n, 7, device="cuda")
    oa, ra, _, _ = env_a.step([big[:, 1:6] for _ in range(3)])                  # strided views
    ob, rb, _, _ = env_b.step([big[:, 1:6].contiguous() for _ in range(3)])
    for x, y in zip(oa + ra, ob + rb):
        assert torch.equal(x, y)


@pytest.mark.parametrize("n", [2048, 70001])
def test_host_buffers_path_equals_device_path(n):
    """NumPy in -> NumPy out through mpe_step_host equals the CUDA-tensor path bit for bit (70001 worlds take
    the chunk-pipelined route: 4 ranges over two internal streams, ragged last range)"""
    import os
    os.environ["MPE_B200_HOST_CHUNK_MIN"] = "16384"      # read once by the library, before its first host step
    env_a = make_product_env("simple_world_comm", num_envs=n)
    env_b = make_product_env("simple_world_comm", num_envs=n)
    env_a.reset()
    env_b.reset()
    env_b.world.native.agent_pv.copy_(env_a.world.native.agent_pv)
    env_b.world.native.lm_p.copy_(env_a.world.native.lm_p)
    rng = np.random.RandomState(3)
    act = random_actions(env_a.world.native.act_dims, n, rng).astype(np.float32)
    acts = split_cols(act, env_a.world.native.act_dims)
    for _ in range(3):
        oa, ra, da, _ = env_a.step([torch.as_tensor(np.ascontiguousarray(a), device="cuda") for a in acts])
        ob, rb, db, _ = env_b.step([np.ascontiguousarray(a) for a in acts])
        assert isinstance(ob[0], np.ndarray) and ob[0].shape == (n, 34)
        for x, y in zip(oa, ob):
            assert np.array_equal(x.cpu().numpy(), y)
        for x, y in zip(ra, rb):
            assert np.array_equal(x.cpu().numpy(), y)
        assert not any(d.any() for d in db)


def test_step_async_matches_step_and_interleaves_two_envs():
    """step_async / step_wait == step, and two envs can be in flight at once (the use case: overlap the
    transfers of one batch with host work on another)"""
    n = 4096
    envs = [make_product_env("simple_tag", num_envs=n, seed=s) for s in (1, 2)]
    refs = [make_product_env("simple_tag", num_envs=n, seed=s) for s in (1, 2)]
    for e in envs + refs:
        e.reset()
    rng = np.random.RandomState(0)
    for t in range(3):
        acts = [[np.ascontiguousarray(a) for a in split_cols(random_actions(e.world.native.act_dims, n, rng).astype(np.float32),
                                                             e.world.native.act_dims)] for e in envs]
        for e, a in zip(envs, acts):
            e.step_async(a)                       # both steps are enqueued before either is collected
        outs = [e.step_wait() for e in envs]
        for r, a, (obs_n, rew_n, done_n, info_n) in zip(refs, acts, outs):
            ro, rr, rd, _ = r.step(a)
            for x, y in zip(obs_n + rew_n, ro + rr):
                assert isinstance(x, np.ndarray) and np.array_equal(x, y)
    with pytest.raises(RuntimeError):
        envs[0].step_wait()


_ALT_SCRIPT = r"""
import sys, numpy as np, torch
sys.path.insert(0, %(root)r); sys.path.insert(0, %(root)r + "/tests")
from helpers import make_product_env
out = {}
for tag, n in (("simple_spread_n3", 5003), ("simple_spread_n6", 2049), ("simple_tag", 4097), ("simple_world_comm", 3001),
               ("simple_reference", 1000), ("simple_crypto", 999), ("simple_speaker_listener", 64), ("simple_push", 33),
               ("simple_spread_n4", 2081), ("simple_tag_2v1", 1055), ("simple_tag_4v2", 3093)):
    env = make_product_env(tag, num_envs=n, seed=21)
    env.reset()
    g = torch.Generator(device="cuda").manual_seed(4)
    nw = env.world.native
    for t in range(3):
        acts = []
        for d, ag in zip(nw.act_dims, env.agents):
            parts = [torch.softmax(3 * torch.randn(n, 5, device="cuda", generator=g), 1)] if ag.movable else []
            if d - (5 if ag.movable else 0) > 0:
                parts.append(torch.rand(n, d - (5 if ag.movable else 0), device="cuda", generator=g))
            acts.append(torch.cat(parts, 1).contiguous())
        obs_n, rew_n, done_n, _ = env.step(acts)
    out[tag + "_obs"] = torch.cat(obs_n, 1).cpu().numpy()
    out[tag + "_rew"] = torch.stack(rew_n).cpu().numpy()
    out[tag + "_done"] = torch.stack(done_n).cpu().numpy()
    out[tag + "_pv"] = nw.agent_pv.cpu().numpy()
    out[tag + "_comm"] = nw.comm.cpu().numpy()
    if env._last_out.info is not None:
        out[tag + "_info"] = env._last_out.info.cpu().numpy()
np.savez(sys.argv[1], **out)
"""


ALT_KERNELS = {
    "general_kernel_instead_of_hot": {"MPE_B200_HOT": "0"},     # the un-specialised fused step for every tile
    "low_register_build": {"MPE_B200_DENSE": "1"},                # the 80-register HOT variant (tag family, spread N=4)
    # the default kernels (HOT whole tiles, general-kernel tails) in 3- and 4-warp blocks instead of 1-warp blocks:
    # per-warp shared-memory offsets and partial last blocks
    "three_warp_blocks": {"MPE_B200_WPB": "3"},
    "four_warp_blocks": {"MPE_B200_WPB": "4"},
    "four_warp_blocks_low_register_build": {"MPE_B200_WPB": "4", "MPE_B200_DENSE": "1"},
}


@pytest.mark.parametrize("variant", list(ALT_KERNELS))
def test_alternative_step_kernels_are_bit_identical(tmp_path, variant):
    """The default fused step runs whole tiles on the HOT specialisation and ragged tails on the general kernel.
    MPE_B200_HOT=0 runs everything on the general kernel.  Three consecutive steps of eleven programs (the four with an
    80-register build among them) with ragged batch sizes must agree bit for bit."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    res = {}
    for mode in ("0", "1"):
        path = str(tmp_path / ("alt%s.npz" % mode))
        env = dict(os.environ)
        for k in ("MPE_B200_HOT", "MPE_B200_DENSE", "MPE_B200_WPB"):
            env.pop(k, None)
        if mode == "1":
            env.update(ALT_KERNELS[variant])
        subprocess.run([sys.executable, "-c", _ALT_SCRIPT % {"root": root}, path], check=True, env=env, timeout=900)
        res[mode] = dict(np.load(path))
    assert set(res["0"]) == set(res["1"]) and len(res["0"]) >= 55
    for k in res["0"]:
        assert np.array_equal(res["0"][k], res["1"][k]), k
