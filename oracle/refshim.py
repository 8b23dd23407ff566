"""TEST INFRASTRUCTURE ONLY -- never imported by the product package.

Imports the *unmodified* Python reference from /root/reference in this container so that
(a) the C oracle restatement (oracle/mpe_oracle.c) can be pinned against it and
(b) golden input/output fixtures can be generated (tests/golden/make_golden.py).

The reference needs `gym` (not installed) and the stdlib module `imp` (removed in 3.12) only for
type scaffolding, never for arithmetic; the stubs below provide exactly the names it touches
(SURVEY.md section 8(c)):  gym.Env, gym.Space, gym.spaces.{Discrete,Box,Tuple,prng},
gym.envs.registration.{register,EnvSpec}, imp.load_source.

/root/reference does not exist on the GPU box: nothing under tests/ -m gpu, smoke() or bench.py
may import this module.
"""
import importlib.machinery
import importlib.util
import os
import sys
import types

REFERENCE_ROOT = os.environ.get("MPE_REFERENCE_ROOT", "/root/reference")


def available():
    return os.path.isdir(os.path.join(REFERENCE_ROOT, "multiagent"))


def _install_stubs():
    import numpy as np

    if "gym" not in sys.modules:
        gym = types.ModuleType("gym")

        class Env(object):
            pass

        class Space(object):
            pass

        gym.Env = Env
        gym.Space = Space
        spaces = types.ModuleType("gym.spaces")

        class Discrete(Space):
            def __init__(self, n):
                self.n = n

        class Box(Space):
            def __init__(self, low, high, shape=None, dtype=None):
                self.low, self.high, self.shape, self.dtype = low, high, shape, dtype

        class Tuple(Space):
            def __init__(self, spaces_):
                self.spaces = spaces_

        spaces.Discrete, spaces.Box, spaces.Tuple = Discrete, Box, Tuple
        prng = types.ModuleType("gym.spaces.prng")
        prng.np_random = np.random.RandomState(0)
        spaces.prng = prng
        envs = types.ModuleType("gym.envs")
        registration = types.ModuleType("gym.envs.registration")
        registration.register = lambda *a, **k: None

        class EnvSpec(object):
            pass

        registration.EnvSpec = EnvSpec
        envs.registration = registration
        gym.spaces, gym.envs = spaces, envs
        sys.modules.update({
            "gym": gym, "gym.spaces": spaces, "gym.spaces.prng": prng,
            "gym.envs": envs, "gym.envs.registration": registration,
        })
    if "imp" not in sys.modules:
        imp = types.ModuleType("imp")

        def load_source(name, pathname):
            loader = importlib.machinery.SourceFileLoader(name or "_ref_scenario", pathname)
            spec = importlib.util.spec_from_loader(loader.name, loader)
            mod = importlib.util.module_from_spec(spec)
            loader.exec_module(mod)
            return mod

        imp.load_source = load_source
        sys.modules["imp"] = imp


def import_reference():
    """Returns (make_env, multiagent) of the real reference.  Raises if it is not mounted."""
    if not available():
        raise RuntimeError("reference not mounted at %s" % REFERENCE_ROOT)
    os.environ["SUPPRESS_MA_PROMPT"] = "1"
    _install_stubs()
    # the product ships a drop-in package that is also called `multiagent`; make sure the
    # reference's own package wins inside this (test-only) process
    for k in [k for k in sys.modules if k == "multiagent" or k.startswith("multiagent.") or k == "make_env"]:
        del sys.modules[k]
    if REFERENCE_ROOT in sys.path:
        sys.path.remove(REFERENCE_ROOT)
    sys.path.insert(0, REFERENCE_ROOT)
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        import multiagent  # noqa: F401  (the reference's)
        try:
            import make_env as ref_make_env
            make_env = ref_make_env.make_env
        except ImportError:
            # a `pip install --target` of the reference ships the `multiagent` package but not the top-level
            # make_env.py; this is the body of make_env.py:36-43 expressed through the package's own classes
            def make_env(scenario_name, benchmark=False):
                from multiagent.environment import MultiAgentEnv
                import multiagent.scenarios as scenarios
                scenario = scenarios.load(scenario_name + ".py").Scenario()
                world = scenario.make_world()
                if benchmark:
                    return MultiAgentEnv(world, scenario.reset_world, scenario.reward, scenario.observation,
                                         scenario.benchmark_data)
                return MultiAgentEnv(world, scenario.reset_world, scenario.reward, scenario.observation)
    assert os.path.realpath(multiagent.__file__).startswith(os.path.realpath(REFERENCE_ROOT)), multiagent.__file__
    return make_env, multiagent


def make_reference_env(name, n=None):
    """Reference env for `name`; `simple_spread` accepts n (agents = landmarks = n), `simple_tag` a tuple
    (adversaries, good agents, landmarks) and `simple_adversary` n (agents; n - 1 landmarks), by building the
    world test-side with the reference's own property assignments (e.g. simple_spread.py:15-26) and reusing
    its generic reset_world / reward / observation (SURVEY.md 8(c) "N=6 spread")."""
    make_env, multiagent = import_reference()
    if name == "simple_spread" and n not in (None, 3):
        from multiagent.core import World, Agent, Landmark
        from multiagent.environment import MultiAgentEnv
        import multiagent.scenarios as scenarios
        scenario = scenarios.load("simple_spread.py").Scenario()
        world = World()
        world.dim_c = 2
        world.collaborative = True
        world.agents = [Agent() for _ in range(n)]
        for i, agent in enumerate(world.agents):
            agent.name = "agent %d" % i
            agent.collide = True
            agent.silent = True
            agent.size = 0.15
        world.landmarks = [Landmark() for _ in range(n)]
        for i, landmark in enumerate(world.landmarks):
            landmark.name = "landmark %d" % i
            landmark.collide = False
            landmark.movable = False
        scenario.reset_world(world)
        return MultiAgentEnv(world, scenario.reset_world, scenario.reward, scenario.observation,
                             scenario.benchmark_data)
    if name == "simple_tag" and isinstance(n, tuple):
        # (num_adversaries, num_good_agents, num_landmarks) other than the hard-coded 3/1/2: the world is built
        # test-side with the reference's own property assignments (simple_tag.py:16-33); its reset_world / reward /
        # observation / benchmark_data are generic over world.agents / world.landmarks and are reused unchanged
        from multiagent.core import World, Agent, Landmark
        from multiagent.environment import MultiAgentEnv
        import multiagent.scenarios as scenarios
        scenario = scenarios.load("simple_tag.py").Scenario()
        n_adv, n_good, n_lm = n
        world = World()
        world.dim_c = 2
        world.agents = [Agent() for _ in range(n_adv + n_good)]
        for i, agent in enumerate(world.agents):
            agent.name = "agent %d" % i
            agent.collide = True
            agent.silent = True
            agent.adversary = i < n_adv
            agent.size = 0.075 if agent.adversary else 0.05
            agent.accel = 3.0 if agent.adversary else 4.0
            agent.max_speed = 1.0 if agent.adversary else 1.3
        world.landmarks = [Landmark() for _ in range(n_lm)]
        for i, landmark in enumerate(world.landmarks):
            landmark.name = "landmark %d" % i
            landmark.collide = True
            landmark.movable = False
            landmark.size = 0.2
            landmark.boundary = False
        scenario.reset_world(world)
        return MultiAgentEnv(world, scenario.reset_world, scenario.reward, scenario.observation, scenario.benchmark_data)
    if name == "simple_adversary" and n not in (None, 3):
        # n agents (one adversary) and n - 1 landmarks, built test-side with the reference's own property assignments
        # (simple_adversary.py:8-31); its reset_world / reward / observation / benchmark_data are generic over
        # world.num_agents / world.agents / world.landmarks and are reused unchanged
        from multiagent.core import World, Agent, Landmark
        from multiagent.environment import MultiAgentEnv
        import multiagent.scenarios as scenarios
        scenario = scenarios.load("simple_adversary.py").Scenario()
        world = World()
        world.dim_c = 2
        world.num_agents = n
        world.agents = [Agent() for _ in range(n)]
        for i, agent in enumerate(world.agents):
            agent.name = "agent %d" % i
            agent.collide = False
            agent.silent = True
            agent.adversary = i < 1
            agent.size = 0.15
        world.landmarks = [Landmark() for _ in range(n - 1)]
        for i, landmark in enumerate(world.landmarks):
            landmark.name = "landmark %d" % i
            landmark.collide = False
            landmark.movable = False
            landmark.size = 0.08
        scenario.reset_world(world)
        return MultiAgentEnv(world, scenario.reset_world, scenario.reward, scenario.observation, scenario.benchmark_data)
    return make_env(name, benchmark=(name not in ("simple", "simple_push", "simple_reference",
                                                  "simple_speaker_listener")))
