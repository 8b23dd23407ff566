"""CPU checks that tie the two-hidden-layer actor's host side to the built library: every one of its 170 kernels (17
programs x H = 32, 64 x the four MADDPG forms, and 17 programs x MAPPO's two forms at H = 64) is compiled for the block
size the test mirror (mlp_programs.mlp_block_cap) expects, read from the kernel's launch bounds in libmpe_b200.so; and
the six entry points refuse what they can refuse without a device with the return codes they always had.  Also: the
programs with step, rollout and 80-register step kernels in the library are the ones the GPU tests parametrize."""
import os
import re
import shutil
import subprocess

import pytest

from helpers import PROGRAM_TAGS, STEP_DENSE_TAGS, TYPE_TAGS, make_product_env
from mlp_programs import PROGRAMS, mlp_block_cap

pytest.importorskip("torch")

# kernel name -> (episodes, categorical, mappo)
FORMS = {"mlp_rollout": (False, False, False), "mlp_episode": (True, False, False),
         "mlp_categorical": (False, True, False), "mlp_categorical_episode": (True, True, False),
         "mappo": (False, True, True), "mappo_episode": (True, True, True)}


def cuobjdump():
    """cuobjdump of the toolkit whose nvcc builds the library (the Makefile's NVCC, else nvcc on PATH)"""
    nvcc = shutil.which(os.environ.get("NVCC", "nvcc"))
    for d in ([os.path.dirname(os.path.realpath(nvcc))] if nvcc else []) + \
            [os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin")]:
        if os.access(os.path.join(d, "cuobjdump"), os.X_OK):
            return os.path.join(d, "cuobjdump")
    pytest.skip("no CUDA toolkit (cuobjdump) to read the library with")


def max_threads_per_kernel(lib_path):
    """mangled kernel name -> EIATTR_MAX_THREADS (x) of its .nv.info section in `cuobjdump -elf`"""
    text = subprocess.run([cuobjdump(), "-elf", lib_path], capture_output=True, text=True, check=True).stdout
    out, cur, attr = {}, None, False
    for ln in text.splitlines():
        if ln.startswith("."):
            cur = ln[len(".nv.info."):] if ln.startswith(".nv.info.") else None
            attr = False
        elif cur and "Attribute:" in ln:
            attr = ln.split()[-1] == "EIATTR_MAX_THREADS"
        elif cur and attr and ln.strip().startswith("Value:"):
            out[cur] = int(ln.split()[1], 16)
            attr = False
    return out


def test_launch_bounds_are_the_mirrored_caps():
    from multiagent_particle_envs_b200 import _lib
    threads = max_threads_per_kernel(_lib.LIB_PATH)
    names = list(threads)
    demangled = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True,
                               check=True).stdout.split("\n")
    seen = {}
    for mangled, nm in zip(names, demangled):
        m = re.match(r"void mpe::mpe_policy_(mlp_rollout|mlp_episode|mlp_categorical|mlp_categorical_episode)_kernel"
                     r"<mpe::(.+), (\d+)>\(", nm)
        if m:
            seen[(TYPE_TAGS[m.group(2)], int(m.group(3))) + FORMS[m.group(1)]] = threads[mangled]
        m = re.match(r"void mpe::mpe_policy_(mappo|mappo_episode)_kernel<mpe::(.+?)\s*>\(", nm)
        if m:                                        # MAPPO's actor: H = 64 only
            seen[(TYPE_TAGS[m.group(2)], 64) + FORMS[m.group(1)]] = threads[mangled]
    assert len(seen) == 170 and {k[0] for k in seen} == set(PROGRAMS)
    assert sum(k[4] for k in seen) == 34
    want = {(tag, H, e, c, mp): 32 * mlp_block_cap(tag, H, e, c, mp) for tag, H, e, c, mp in seen}
    assert seen == want


def test_every_step_program_is_in_the_test_tables():
    """The programs with a fused step (mpe_kernel) and an open-loop rollout (mpe_rollout_kernel) in libmpe_b200.so are
    exactly helpers.PROGRAM_TAGS, which the step, rollout and reset tests run; those with the 80-register HOT build
    (mpe_kernel<P, kFusedStep, true, true>) are exactly helpers.STEP_DENSE_TAGS, which the oracle test runs at sizes
    that select it.  A program or a low-register build added without a place in those tests fails here."""
    from multiagent_particle_envs_b200 import _lib
    names = list(max_threads_per_kernel(_lib.LIB_PATH))
    demangled = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True,
                               check=True).stdout.split("\n")
    step, rollout, dense = set(), set(), set()
    for nm in demangled:
        m = re.match(r"void mpe::mpe_kernel<mpe::(.+), (\d), (true|false), (true|false)>\(", nm)
        if m:
            step.add(TYPE_TAGS[m.group(1)])
            if (m.group(2), m.group(3), m.group(4)) == ("0", "true", "true"):      # kFusedStep, HOT, DENSE
                dense.add(TYPE_TAGS[m.group(1)])
        m = re.match(r"void mpe::mpe_rollout_kernel<mpe::(.+?)\s*>\(", nm)
        if m:
            rollout.add(TYPE_TAGS[m.group(1)])
    assert step == rollout == set(PROGRAM_TAGS)
    assert dense == set(STEP_DENSE_TAGS)


# ---- return codes without a device ---------------------------------------------------------------------------------
ENTRY_POINTS = ("mpe_rollout_policy_mlp", "mpe_rollout_policy_mlp_categorical", "mpe_rollout_policy_mlp_episodes",
                "mpe_rollout_policy_mlp_categorical_episodes", "mpe_rollout_policy_mappo",
                "mpe_rollout_policy_mappo_episodes")
# MAPPO's entry points -> the categorical form whose return codes they give
MAPPO_BASE = {"mpe_rollout_policy_mappo": "mpe_rollout_policy_mlp_categorical",
              "mpe_rollout_policy_mappo_episodes": "mpe_rollout_policy_mlp_categorical_episodes"}
BAD_ARG, NO_DEVICE = -1, -5


def _call(name, handle, steps=4, weights=True, hidden=32):
    """`name` with aligned dummy pointers (every probe returns before one is used), hidden width `hidden`, `steps` steps
    (the episode length in the episode forms, of one episode) and null weight arrays unless `weights`"""
    from multiagent_particle_envs_b200 import _lib
    lib = _lib.load()
    argtypes = _lib._SIGNATURES[name][1]
    per_agent = _lib.ptr_array([256] * _lib.MPE_MAX_AGENTS)
    args = [256 if t is _lib._P else per_agent if t is _lib._PP else 1 if t.__name__ == "c_int" else 0 for t in argtypes]
    args[0], args[-1] = handle, None
    args[5:11] = [per_agent if weights else None] * 6
    args[11], args[12] = hidden, steps
    return getattr(lib, name)(*args)


def test_entry_point_return_codes_without_a_device():
    """the single-episode forms refuse a negative n_steps and null weight arrays before they ask for the device; the
    episode forms ask for the device first; MAPPO's entry points, at either width, answer as the categorical ones"""
    shapes = make_product_env("simple_spread_n3", num_envs=64).world.native_shapes()   # device-less handle
    handle = shapes.handle          # `shapes` owns it: the handle stays live while the test holds `shapes`
    for name in ENTRY_POINTS:
        episodes = name.endswith("_episodes")
        for hidden in (32, 64):
            probes = [dict(handle=None), dict(handle=handle, steps=-1), dict(handle=handle, weights=False),
                      dict(handle=handle)]
            want = [BAD_ARG, NO_DEVICE if episodes else BAD_ARG, NO_DEVICE if episodes else BAD_ARG, NO_DEVICE]
            for kw, w in zip(probes, want):
                got = _call(name, hidden=hidden, **kw)
                assert got == w, (name, hidden, kw)
                if name in MAPPO_BASE:
                    assert got == _call(MAPPO_BASE[name], hidden=hidden, **kw), (name, hidden, kw)
