"""Pins the CPU oracle (oracle/mpe_oracle.c) against the reference's own outputs.

The fixtures in tests/golden/ were produced by running the unmodified Python reference
(tests/golden/make_golden.py); kat.npz additionally matches the known-answer literals recorded in
SURVEY.md section 8(c).  fp64 oracle: agreement to ~1e-12; fp32 oracle: within the north-star
tolerance (rtol 1e-5, atol 1e-6 per step)."""
import numpy as np
import pytest

from helpers import CONFIGS, descriptor, explain_flag_mismatches, load_golden, step_flags
from oracle import Oracle

TAGS = list(CONFIGS)
NP_PORT_TAGS = list(CONFIGS)


def goal_of(g):
    return g["goal"] if "goal" in g and g["goal"].shape[1] > 0 else None


# worlds the reference's callbacks support but its make_world hard-codes away (built test-side, oracle/refshim.py)
VARIANT_TAGS = ["simple_tag_1v1", "simple_tag_4v2", "simple_tag_6v2", "simple_tag_2v1", "simple_spread_n2",
                "simple_spread_n4", "simple_spread_n5", "simple_adversary_n4"]


@pytest.mark.parametrize("tag", TAGS + ["simple_tag_force_discrete", "simple_tag_discrete_input"] + VARIANT_TAGS)
def test_oracle_f64_trajectory_matches_reference(tag):
    g = load_golden(tag)
    base = tag if tag in VARIANT_TAGS else ("simple_tag" if tag.startswith("simple_tag") else tag)
    orc = Oracle(descriptor(base), "f64")
    assert orc.obs_dims == list(g["prop_obs_dims"]) and orc.act_dims == list(g["prop_act_dims"])
    flags = step_flags(g) | (4 if int(g.get("discrete_input", 0)) else 0)      # MPE_FLAG_DISCRETE_ACTION_INPUT
    pv, comm, lm = g["pv0"], g["comm0"], g["lm"]
    W, T = g["act"].shape[:2]
    for t in range(T):
        pv, comm, obs, rew, done, info = orc.step(pv, lm, comm, g["act"][:, t], flags, goal=goal_of(g))
        np.testing.assert_allclose(pv, g["pv"][:, t], rtol=1e-11, atol=1e-13)
        np.testing.assert_allclose(comm, g["comm"][:, t], rtol=0, atol=0)
        np.testing.assert_allclose(obs, g["obs"][:, t], rtol=1e-11, atol=1e-13)
        np.testing.assert_allclose(rew, g["rew"][:, t], rtol=1e-11, atol=1e-12)
        assert np.array_equal(done, g["done"][:, t])
        if orc.info_dim:
            np.testing.assert_allclose(info, g["info"][:, t], rtol=1e-11, atol=1e-12)


@pytest.mark.parametrize("tag", TAGS)
def test_oracle_f32_single_step_within_tolerance(tag):
    """state re-injected every step (BASELINE.md section 4.4)"""
    g = load_golden(tag)
    orc = Oracle(descriptor(tag), "f32")
    flags = step_flags(g)
    W, T = g["act"].shape[:2]
    flipped = 0
    for t in range(T):
        pv_in = g["pv0"] if t == 0 else g["pv"][:, t - 1]
        comm_in = g["comm0"] if t == 0 else g["comm"][:, t - 1]
        pv, comm, obs, rew, done, info = orc.step(pv_in, g["lm"], comm_in, g["act"][:, t], flags, goal=goal_of(g))
        np.testing.assert_allclose(pv, g["pv"][:, t], rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(obs, g["obs"][:, t], rtol=1e-5, atol=1e-6)
        assert np.array_equal(done, g["done"][:, t])
        # rewards / benchmark_data contain contact indicators: every mismatch must be a flipped indicator whose
        # fp64 distance is within 2e-6 of its threshold (helpers.explain_flag_mismatches)
        flipped += explain_flag_mismatches(tag, rew, g["rew"][:, t], info if orc.info_dim else None,
                                           g["info"][:, t] if orc.info_dim else None, g["pv"][:, t], g["lm"],
                                           g["prop_agent_size"], g["prop_landmark_size"], atol=2e-6)
    assert flipped <= max(2, W * T // 200), flipped      # and they are rare


def test_known_answers_of_survey():
    """literal KATs from SURVEY.md 8(c) (np.random.seed(0); reset; two one-hot steps)"""
    k = dict(np.load(__import__("os").path.join(__import__("helpers").GOLDEN, "kat.npz")))
    np.testing.assert_allclose(k["simple/pv0"][0, :2], [-0.15269040132219058, 0.29178822613331223], rtol=0, atol=0)
    np.testing.assert_allclose(k["simple/pv"][0], [-0.2901904013221906, 0.29178822613331223, -0.875, 0.0], rtol=1e-15)
    np.testing.assert_allclose(k["simple/obs"], [-0.875, 0, 0.16536482384757561, 0.4917577754308473], rtol=1e-15)
    np.testing.assert_allclose(k["simple/rew"], [-0.2691712346628354], rtol=1e-15)
    np.testing.assert_allclose(k["simple_spread/rew"], [-7.463450752813834] * 3, rtol=1e-15)
    np.testing.assert_allclose(k["simple_spread/pv"][0], [0.27358912218786463, 0.8511932765853221, 0.875, 0], rtol=1e-15)
    assert np.all(k["simple_spread/obs"][14:18] == 0)
    np.testing.assert_allclose(k["simple_tag/pv"][0, :3], [0.21858912218786464, 0.8511932765853221, 0.5250000000000001], rtol=1e-15)
    assert np.all(k["simple_tag/rew"] == 0)
    for name, tag in (("simple", "simple"), ("simple_spread", "simple_spread_n3"), ("simple_tag", "simple_tag"),
                      ("simple_world_comm", "simple_world_comm")):
        orc = Oracle(descriptor(tag), "f64")
        flags = step_flags(tag)
        pv, comm = k[name + "/pv0"][None], k[name + "/comm0"][None]
        for _ in range(2):
            pv, comm, obs, rew, done, info = orc.step(pv, k[name + "/lm"][None], comm, k[name + "/act"][None], flags)
        np.testing.assert_allclose(pv[0], k[name + "/pv"], rtol=1e-12, atol=1e-60)
        np.testing.assert_allclose(obs[0], k[name + "/obs"], rtol=1e-12, atol=1e-60)
        np.testing.assert_allclose(rew[0], k[name + "/rew"], rtol=1e-12, atol=1e-15)
        assert np.array_equal(done[0], k[name + "/done"])


@pytest.mark.parametrize("tag", NP_PORT_TAGS)
def test_numpy_port_matches_reference(tag):
    """oracle/np_port.py (the per-world NumPy stand-in for the reference's own path that bench.py times)"""
    import np_port
    g = load_golden(tag)
    spec = np_port.WorldSpec(descriptor(tag))
    shared = bool(int(g["prop_shared_reward"]))
    W, T = g["act"].shape[:2]
    adims = [int(x) for x in g["prop_act_dims"]]
    for w in range(min(W, 4)):
        pos = np.concatenate([g["pv0"][w][:, 0:2], g["lm"][w]]).copy()
        vel = g["pv0"][w][:, 2:4].copy()
        comm = g["comm0"][w].copy()
        for t in range(T):
            acts, c0 = [], 0
            for dmn in adims:
                acts.append(g["act"][w, t, c0:c0 + dmn])
                c0 += dmn
            goal = [int(x) for x in g["goal"][w]] if "goal" in g and g["goal"].shape[1] else None
            obs, rew, done = np_port.env_step(spec, pos, vel, comm, acts, shared, goal=goal)
            np.testing.assert_allclose(np.concatenate(obs), g["obs"][w, t], rtol=1e-11, atol=1e-13)
            np.testing.assert_allclose(np.array(rew, dtype=np.float64), g["rew"][w, t], rtol=1e-11, atol=1e-12)
            np.testing.assert_allclose(pos[:spec.A], g["pv"][w, t][:, 0:2], rtol=1e-11, atol=1e-13)
            assert not any(done)
