"""CPU checks of env.compute_gae (mpe_gae): the float32 mirror the GPU tests judge the kernel by, run in float64, equals a
literal float64 transcription of MAPPO's compute_returns loop; every refusal compute_gae makes before anything runs;
the C ABI and its device-less return codes in their documented order; and the launch bounds of the three kernels."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

from gae_helpers import gae_mirror, mappo_returns, normalize_mirror, seeded_inputs
from helpers import make_product_env
from test_cpu_mlp_block_table import max_threads_per_kernel

torch = pytest.importorskip("torch")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("per_agent", [None, False, True], ids=["no_value_norm", "shared", "per_agent"])
@pytest.mark.parametrize("episodes", [1, 4])
@pytest.mark.parametrize("bootstrap", [True, False])
def test_the_mirror_in_float64_is_mappos_loop(bootstrap, episodes, per_agent):
    """the mirror's operation order in float64 against MAPPO's compute_returns, one buffer per episode"""
    T, n, N = 24, 3, 37
    rew, val, final, vn = seeded_inputs(T, n, N, episodes, seed=episodes, per_agent_norm=bool(per_agent))
    vn = None if per_agent is None else vn
    L = None if episodes == 1 else T // episodes
    ret, adv, _ = gae_mirror(rew, val, final, 0.99, 0.95, L, bootstrap, vn, dtype=np.float64)
    want = mappo_returns(rew, val, final, 0.99, 0.95, L, bootstrap, vn)
    np.testing.assert_allclose(ret, want, rtol=0, atol=1e-12 * (1 + np.abs(want).max()))
    # gae + dv is the return: the advantages are MAPPO's returns - denormalize(value_preds)
    v, vn = val.astype(np.float64), None if vn is None else vn.astype(np.float64)
    dv = v if vn is None else \
        v * (vn[1] if vn.ndim == 1 else vn[:, 1].reshape(n, 1)) + (vn[0] if vn.ndim == 1 else vn[:, 0].reshape(n, 1))
    np.testing.assert_allclose(adv, want - dv, rtol=0, atol=1e-11 * (1 + np.abs(want).max()))


def test_the_float32_mirror_is_within_its_bound_of_mappos_loop():
    """the running error bound of the float32 mirror holds against the float64 loop (the bound is derived, so the
    margin is what it is; the check is that it is never exceeded)"""
    rew, val, final, vn = seeded_inputs(50, 3, 200, 2, seed=7, per_agent_norm=True)
    ret, _, bound = gae_mirror(rew, val, final, 0.99, 0.95, 25, True, vn)
    want = mappo_returns(rew, val, final, 0.99, 0.95, 25, True, vn)
    err = np.abs(ret.astype(np.float64) - want)
    assert (err <= bound + 1e-12 * (1 + np.abs(want))).all()
    assert err.max() > 0 and bound.max() < 1e-4 * np.abs(want).max()


def test_normalize_mirror_is_ppos_step():
    """(A - mean) / (std + 1e-5) with NumPy's population std"""
    adv = np.random.RandomState(3).standard_normal((10, 3, 7)).astype(np.float32)
    a64 = adv.astype(np.float64)
    got = normalize_mirror(adv, a64.mean(), a64.std())
    np.testing.assert_allclose(got, (a64 - np.nanmean(a64)) / (np.nanstd(a64) + 1e-5), rtol=1e-6, atol=1e-6)


# ---- refusals ----------------------------------------------------------------------------------------------------------
def test_refuses_a_non_batched_env():
    env = make_product_env("simple_spread_n3")
    x = torch.zeros(4, 3, 1)
    with pytest.raises(ValueError, match="batched"):
        env.compute_gae(x, x, x[0])


def _good(T=4, n=3, N=8):
    z = lambda *s: torch.zeros(*s, dtype=torch.float32)   # noqa: E731
    return z(T, n, N), z(T, n, N), z(n, N)


@pytest.mark.parametrize("case,match", [
    (dict(rewards=np.zeros((4, 3, 8), dtype=np.float32)), "T >= 1"),
    (dict(rewards=torch.zeros(4, 3, 8, dtype=torch.float64)), "contiguous float32"),
    (dict(rewards=torch.zeros(8, 3, 4).transpose(0, 2)), "contiguous"),
    (dict(rewards=torch.zeros(4, 3, 9)), "shape"),
    (dict(rewards=torch.zeros(0, 3, 8)), "T >= 1"),
    (dict(rewards=torch.zeros(3, 8)), "T >= 1"),
    (dict(values=torch.zeros(5, 3, 8)), "values must have shape"),
    (dict(values=torch.zeros(4, 3, 8, dtype=torch.float16)), "values must be a contiguous"),
    (dict(values=torch.zeros(4, 8, 3).transpose(1, 2)), "values must be a contiguous"),
    (dict(final_values=torch.zeros(2, 3, 8)), "final_values must have shape"),
    (dict(final_values=torch.zeros(3, 8), episode_length=2), r"final_values must have shape \(2, 3, 8\)"),
    (dict(final_values=torch.zeros(3, 8), episode_length=4), r"final_values must have shape \(1, 3, 8\)"),
    (dict(final_values=torch.zeros(3, 8, dtype=torch.float64)), "final_values must be a contiguous"),
    (dict(final_values=torch.zeros(3, 8), bootstrap=False, episode_length=2), "final_values must have shape"),
    (dict(final_values=None), "needs final_values"),
    (dict(episode_length=3), "episode_length"),
    (dict(episode_length=0), "episode_length"),
    (dict(value_norm=torch.zeros(3)), "value_norm must have shape"),
    (dict(value_norm=torch.zeros(2, 2)), "value_norm must have shape"),
    (dict(value_norm=torch.zeros(3, 2, dtype=torch.float64)), "value_norm must be a contiguous"),
    (dict(value_norm=[0.0, 1.0]), "value_norm must be a contiguous"),
    (dict(gamma=1.5), "gamma"),
    (dict(gamma=-0.1), "gamma"),
    (dict(gae_lambda=float("nan")), "gae_lambda"),
    (dict(gae_lambda=float("inf")), "gae_lambda"),
])
def test_refusals(case, match):
    """each refusal on otherwise valid CPU tensors: every check but the device's comes before the env is bound"""
    env = make_product_env("simple_spread_n3", num_envs=8)
    rew, val, fin = _good()
    kw = dict(rewards=rew, values=val, final_values=fin)
    kw.update(case)
    with pytest.raises(ValueError, match=match):
        env.compute_gae(**kw)


def test_refuses_host_tensors_before_binding_the_world():
    """tensors off the env's device are refused before the world state is allocated: the env stays unbound"""
    env = make_product_env("simple_spread_n3", num_envs=8)
    rew, val, fin = _good()
    with pytest.raises(ValueError, match="rewards must be a CUDA tensor"):
        env.compute_gae(rew, val, fin)
    assert env.world._native is None


# ---- the C ABI ---------------------------------------------------------------------------------------------------------
BAD_ARG, NO_DEVICE = -1, -5


def test_entry_points_are_declared_exported_and_bound():
    from multiagent_particle_envs_b200 import _lib
    header = open(os.path.join(ROOT, "include", "mpe_b200.h")).read()
    declared = set(re.findall(r"MPE_API[^;(]*?\b(mpe_[a-z_]+)\s*\(", header))
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in ("mpe_gae", "mpe_gae_workspace_bytes"):
        assert name in declared and name in _lib.EXPORTED_SYMBOLS and hasattr(lib, name), name
    P = _lib._P
    assert _lib._SIGNATURES["mpe_gae"][1] == [P, P, P, P, ctypes.c_int32, ctypes.c_int32, ctypes.c_float,
                                              ctypes.c_float, ctypes.c_uint32, P, P, P, P, ctypes.c_int64, P]
    assert (_lib.GAE_BOOTSTRAP, _lib.GAE_NORMALIZE, _lib.GAE_PER_AGENT_VALUE_NORM) == (1, 2, 4)
    assert _lib.MPE_ABI_VERSION == 1


def _call(handle, steps=4, L=0, gamma=0.99, lam=0.95, flags=3, ptrs=True, vn=None, ws=256, ws_bytes=1 << 20):
    from multiagent_particle_envs_b200 import _lib
    p = 256 if ptrs else None
    return _lib.load().mpe_gae(handle, p, p, p, steps, L, gamma, lam, flags, vn, p, p, ws, ws_bytes, None)


def test_entry_point_return_codes_without_a_device():
    """a null handle and n_steps < 1 before the device; everything else (episode length, gamma, lambda, flags,
    pointers, workspace) after it"""
    shapes = make_product_env("simple_spread_n3", num_envs=64).world.native_shapes()   # device-less handle
    h = shapes.handle
    probes = [dict(handle=None), dict(handle=h, steps=0), dict(handle=h, steps=-3), dict(handle=None, steps=0),
              dict(handle=h, L=3), dict(handle=h, L=-1), dict(handle=h, gamma=1.5), dict(handle=h, lam=float("nan")),
              dict(handle=h, flags=8), dict(handle=h, ptrs=False), dict(handle=h, flags=4), dict(handle=h, vn=257),
              dict(handle=h, ws_bytes=0), dict(handle=h, ws=260), dict(handle=h, ws=264), dict(handle=h)]
    assert [_call(**kw) for kw in probes] == [BAD_ARG] * 4 + [NO_DEVICE] * 12


def test_workspace_bytes():
    """32 bytes of header and one fp64 partial (two doubles) per 128 columns of A * N; a null handle is refused"""
    from multiagent_particle_envs_b200 import _lib
    lib = _lib.load()
    for tag, N, A in (("simple_spread_n3", 64, 3), ("simple_spread_n3", 65553, 3), ("simple", 1000, 1)):
        h = make_product_env(tag, num_envs=N).world.native_shapes().handle
        assert lib.mpe_gae_workspace_bytes(h) == 32 + 16 * ((A * N + 127) // 128)
    assert lib.mpe_gae_workspace_bytes(None) == BAD_ARG


def test_launch_bounds():
    """the scan (with and without the fp64 sums) at 128 threads, the normalisation at 256"""
    from multiagent_particle_envs_b200 import _lib
    threads = max_threads_per_kernel(_lib.LIB_PATH)
    names = list(threads)
    demangled = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True,
                               check=True).stdout.split("\n")
    seen = {nm.split("(")[0]: threads[m] for m, nm in zip(names, demangled) if "mpe_gae" in nm}
    assert seen == {"void mpe::mpe_gae_kernel<false>": 128, "void mpe::mpe_gae_kernel<true>": 128,
                    "mpe::mpe_gae_normalize_kernel": 256}
