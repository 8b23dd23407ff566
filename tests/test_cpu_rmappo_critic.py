"""CPU checks of rMAPPO's recurrent centralized critic (env.rollout_policy(rmappo_actors, T, critic=(base, gru, norm,
v_out)), mpe_critic_gru): its fold and the float64 recipe model without rounding against the unfolded modules, the
critics rmappo_critic_params and rollout_policy refuse, the C ABI and its device-less return codes, and the launch
bounds of the 7 kernels against the mirrored block table."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

from helpers import TYPE_TAGS, make_product_env
from mappo_helpers import FEATURE_NORM, TANH, make_mappo_actors
from rcritic_helpers import H, RCRITIC_PROGRAMS, RCRITIC_WARPS, RecurrentModel, make_rcritic
from rmappo_helpers import make_rmappo_actor, module_step
from test_cpu_mlp_block_table import max_threads_per_kernel

torch = pytest.importorskip("torch")
nn = torch.nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBS, ACT = [18] * 3, [5] * 3            # simple_spread N=3: D = 54


def _params(critic, obs=OBS):
    from multiagent_particle_envs_b200.environment import rmappo_critic_params
    return rmappo_critic_params(critic, obs)


@pytest.mark.parametrize("tanh", [False, True])
@pytest.mark.parametrize("fn", [False, True])
def test_the_fold_and_the_unrounded_model_equal_the_modules(tanh, fn):
    """the folded float64 critic (RecurrentModel without rounding, head [1, 64]) against base -> gru -> norm -> v_out in
    float64, on random share_obs rows and hidden states"""
    critic = make_rcritic(OBS, tanh, fn, device="cpu", eps=1e-3)
    params, got_tanh, got_fn, eps = _params(critic)
    assert (got_tanh, got_fn, eps) == (tanh, fn, 1e-3)
    assert [tuple(t.shape) for t in params] == [(H, 54), (H,), (H, H), (H,), (192, H), (192,), (192, H), (192,),
                                                (1, H), (1,)]
    assert all(t.dtype == torch.float64 for t in params)
    rng = np.random.RandomState(0)
    x, h = rng.randn(512, 54) * 2.0, np.tanh(rng.randn(512, H))
    net = ((FEATURE_NORM if fn else 0) | (TANH if tanh else 0), eps)
    v, hn = RecurrentModel([t.numpy() for t in params], net, tf32=False).step(x, h)
    v64, hn64 = module_step(critic, x, h)
    np.testing.assert_allclose(hn, hn64, rtol=0, atol=1e-10)
    np.testing.assert_allclose(v, v64, rtol=0, atol=1e-10)


def test_shared_lists_are_one_critic_and_distinct_tuples_are_refused():
    a = make_rcritic(OBS, False, True, device="cpu")
    ref = _params(a)[0]
    for form in ([a], [a] * 3):
        assert all(torch.equal(p, q) for p, q in zip(_params(form)[0], ref))
    with pytest.raises(NotImplementedError, match="distinct"):
        _params([a, tuple(list(a)), a])


def _variant(**kw):
    base, gru, norm, head = make_rcritic(OBS, False, True, device="cpu")
    parts = dict(base=base, gru=gru, norm=norm, head=head)
    parts.update(kw)
    return (parts["base"], parts["gru"], parts["norm"], parts["head"])


@pytest.mark.parametrize("critic,match", [
    (_variant(gru=nn.GRU(64, 64, num_layers=2)), "num_layers=1"),
    (_variant(gru=nn.GRU(64, 32)), "nn.GRU\\(64, 64\\)"),
    (_variant(head=nn.Linear(64, 5)), "head"),                                      # not one output
    (_variant(head=nn.Linear(64, 1, bias=False)), "bias"),
    (_variant(norm=nn.LayerNorm(64, eps=1e-3)), "same eps"),
    (_variant(base=make_rmappo_actor(18, 1, False, True, device="cpu")[0]), "expected Linear weights"),   # width != D
    (_variant()[:3] + (_variant()[1],), "head"),
    ([_variant()] * 2, "list of 1 or 3"),
])
def test_refuses_malformed_critics(critic, match):
    with pytest.raises(ValueError, match=match):
        _params(critic)


def test_refusals_without_a_device():
    """the pairings and state arguments rollout_policy refuses before the env is bound"""
    env = make_product_env("simple_spread_n3", num_envs=64)
    rcritic = make_rcritic(OBS, False, True, device="cpu")
    actor = make_rmappo_actor(18, 5, False, True, device="cpu")
    mappo = make_mappo_actors(OBS, ACT, False, True, device="cpu")
    sequential = make_mappo_actors([54], [1], False, True, device="cpu")[0]
    with pytest.raises(NotImplementedError, match="recurrent actor"):
        env.rollout_policy(mappo, 4, action_mode="categorical", critic=rcritic)
    with pytest.raises(NotImplementedError, match="recurrent critic"):
        env.rollout_policy([actor] * 3, 4, action_mode="categorical", critic=sequential)
    for kw in (dict(critic_rnn_states=torch.zeros(64, H)), dict(record_critic_rnn_states=True)):
        for actors, critic in (([actor] * 3, None), (mappo, sequential), (mappo, None)):
            with pytest.raises(ValueError, match="critic_rnn_states"):
                env.rollout_policy(actors, 4, action_mode="categorical", critic=critic, **kw)
    with pytest.raises(ValueError, match="episode_length"):
        env.rollout_policy([actor] * 3, 4, action_mode="categorical", critic=rcritic, episode_length=2,
                           critic_rnn_states=torch.zeros(64, H))
    with pytest.raises(NotImplementedError, match="categorical"):
        env.rollout_policy([actor] * 3, 4, critic=rcritic)


# ---- the C ABI ----------------------------------------------------------------------------------------------------------
BAD_ARG, NO_DEVICE = -1, -5


def test_entry_point_is_declared_exported_and_bound():
    from multiagent_particle_envs_b200 import _lib
    header = open(os.path.join(ROOT, "include", "mpe_b200.h")).read()
    declared = set(re.findall(r"MPE_API[^;(]*?\b(mpe_[a-z_]+)\s*\(", header))
    lib = ctypes.CDLL(_lib.LIB_PATH)
    name = "mpe_critic_gru"
    assert name in declared and name in _lib.EXPORTED_SYMBOLS and hasattr(lib, name)
    P, PP = _lib._P, _lib._PP
    assert _lib._SIGNATURES[name][1] == [P, PP, PP, ctypes.c_int32, ctypes.c_int32] + [P] * 10 + \
        [P, P, P, P, ctypes.c_uint32, ctypes.c_float, P]
    assert _lib.MPE_ABI_VERSION == 1


def _call(handle, steps=4, episode_length=0, weights=True):
    """mpe_critic_gru with aligned dummy pointers (every probe returns before one is used)"""
    from multiagent_particle_envs_b200 import _lib
    lib = _lib.load()
    per_agent = _lib.ptr_array([256] * _lib.MPE_MAX_AGENTS)
    w = [256 if weights else None] * 10
    return lib.mpe_critic_gru(handle, per_agent, per_agent, steps, episode_length, *w, 256, None, 256, 256, 0, 0.0,
                              None)


def test_entry_point_return_codes_without_a_device():
    """a null handle and a negative n_steps before the device; everything else after it"""
    shapes = make_product_env("simple_spread_n3", num_envs=64).world.native_shapes()   # device-less handle
    probes = [dict(handle=None), dict(handle=shapes.handle, steps=-1), dict(handle=shapes.handle, weights=False),
              dict(handle=shapes.handle, episode_length=3), dict(handle=shapes.handle, episode_length=-1),
              dict(handle=shapes.handle)]
    assert [_call(**kw) for kw in probes] == [BAD_ARG, BAD_ARG, NO_DEVICE, NO_DEVICE, NO_DEVICE, NO_DEVICE]


def test_launch_bounds_are_the_mirrored_table():
    """the 7 kernels: one per program of the recurrent actor, every one at RCRITIC_WARPS warps"""
    from multiagent_particle_envs_b200 import _lib
    threads = max_threads_per_kernel(_lib.LIB_PATH)
    names = list(threads)
    demangled = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True,
                               check=True).stdout.split("\n")
    seen = {}
    for mangled, nm in zip(names, demangled):
        m = re.match(r"void mpe::mpe_critic_gru_kernel<mpe::(.+?)\s*>\(", nm)
        if m:
            seen[TYPE_TAGS[m.group(1)]] = threads[mangled]
    assert set(seen) == set(RCRITIC_PROGRAMS) and len(seen) == 7
    assert set(seen.values()) == {32 * RCRITIC_WARPS}


def test_the_shared_memory_figures():
    """the weight set the kernel's static_asserts state: 512 sum(kt1_i) + 29 704 floats"""
    from mlp_programs import shapes_of
    got = {t: 4 * (512 * sum((od + 7) // 8 for od in shapes_of(t)[0]) + 29704) for t in RCRITIC_PROGRAMS}
    assert (got["simple"], got["simple_spread_n3"], got["simple_reference"], got["simple_spread_n6"]) == \
        (120864, 137248, 131104, 180256)
    assert max(got.values()) <= 232448
