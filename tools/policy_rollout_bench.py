#!/usr/bin/env python
"""Closed-loop rollouts: T steps of obs -> per-agent actor -> env.step, as
  (a) ONE launch of the in-kernel rollout (actors evaluated inside the kernel, state and observations in registers):
      --layers 2: Linear-ReLU-Linear-softmax in fp32 (mpe_rollout_policy);
      --layers 3: MADDPG's Linear-ReLU-Linear-ReLU-Linear on the tensor cores in TF32 (mpe_rollout_policy_mlp),
      --explore: with the Gumbel-softmax sample instead of softmax (--layers 3 only);
      --categorical: policy-gradient actions (action_mode="categorical", --layers 3 only): the one-hot vector of the
      arg-max of the logits (--explore: of the Gumbel-perturbed logits) per sub-space, recording the indices and the
      log-probabilities;
      --actor mappo: MAPPO's actor ([LayerNorm] - Linear - Act - LayerNorm - Linear - Act - LayerNorm - Linear, H = 64,
      mpe_rollout_policy_mappo), --categorical and --layers 3 implied; --tanh for Act = Tanh (else ReLU),
      --feature-norm for the input LayerNorm.  The MADDPG categorical kernel is timed in the same run
      ("maddpg_in_kernel"), so the cost of the LayerNorms and the tanh shows;
      --actor rmappo: MAPPO's recurrent actor, one (base, gru, norm, head) tuple shared by every agent (base = the MAPPO
      actor without its last Linear, nn.GRU(64, 64), LayerNorm(64), Linear(64, act_dim); mpe_rollout_policy_gru), with
      the same implied options and --tanh / --feature-norm;
      --critic shared|separated (with --actor mappo): MAPPO's centralized critic ([LayerNorm(D)] - Linear(D, 64) - Act -
      LayerNorm - Linear - Act - LayerNorm - Linear(64, 1) on every agent's observation concatenated, one shared
      module or one per agent) evaluated in the same launch (critic=..., mpe_rollout_policy_mappo_critic), against
      what a trainer does without it: the same call with record_observations=True, then the torch critic over the
      concatenated records ([T N, D]) and the final observations ([N, D]), at torch's default float32 matmul
      precision.  Only these two arms are timed ("in_kernel_critic", "kernel_then_torch_critic");
      --critic recurrent (with --actor rmappo): rMAPPO's recurrent critic, one (base, gru, norm, v_out) tuple on the
      concatenated observations (critic=..., mpe_critic_gru after the rollout).  Three arms are timed in the same run:
      "in_kernel_critic" (the rollout with the critic), "rollout_recording_observations" (the same rollout with
      record_observations=True and no critic: the difference is the critic kernel's own cost) and
      "kernel_then_torch_critic" (that rollout, then the torch critic under no_grad in its fastest form: base over
      [T N, D] in one call, one cuDNN nn.GRU call over the [T, N, 64] sequence, norm and v_out, plus the bootstrap step
      on the returned observations);
      --critic local (with --actor mappo) / recurrent-local (with --actor rmappo): IPPO's local critics
      (centralized_critic=False), each on its agent's own observation -- one shared critic where every agent observes
      alike, else one per agent.  Arms: "in_kernel_local_critic", the same call without a critic
      ("in_kernel_actor_only", recording observations for recurrent-local), that call then the same local critics in
      torch over the records ("kernel_then_torch_local_critic"), and the centralized critic in-kernel on the same
      program where it has a kernel ("in_kernel_centralized_critic"); with --critic local on a program whose agents
      observe alike, also one critic per agent, local and centralized, where they fit ("..._per_agent");
      --separated (with --actor rmappo, simple_speaker_listener): rMAPPO's separated runner, a distinct tuple per agent
      (mpe_rollout_policy_gru_separated, which restages each agent's weights into shared memory at its turn), and with
      --critic recurrent a distinct critic per agent (mpe_critic_gru_separated; the torch arm runs each critic in turn).
      The restaging traffic per step is reported as computed, not measured: blocks x the sum of the agents' fragment
      image bytes (restage_bytes_per_step);
  (b) the same actors as torch modules + env.step, all captured in one CUDA graph (rollout.GraphedRollout); with
      --categorical the graphed policy takes argmax(logits - log(-log u)) per sub-space, its one_hot and
      log_softmax(logits).gather(k) for the log-probabilities.  With --actor rmappo the graphed policy evaluates the
      shared tuple once on every agent's observations stacked (base -> one nn.GRU step from the carried h, kept in a
      graph-resident tensor -> LayerNorm -> head), at float32 matmul precision "highest".
Device time per step of each.  With --layers 3 the actor of agent i has act_dim_i outputs and its action is one
(Gumbel-)softmax per action sub-space (5 movement logits if the agent moves, then dim_c utterance logits if it speaks).
Also the actor's FLOPs per step, computed from the padded shapes the kernel multiplies (2 (K1 H + H H + NOUT H) per
agent and world, K1 = obs_dim and NOUT = act_dim rounded up to 8), the in-kernel rollout's
achieved TFLOP/s (actor FLOPs over the whole step's time: physics, observations and rewards are in that time too),
torch's float32 matmul precision for the graphed loop, and the card's name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def actor_flops_per_step(obs_dims, act_dims, H, n):
    return sum(2 * (((od + 7) // 8 * 8) * H + H * H + ((ad + 7) // 8 * 8) * H) for od, ad in zip(obs_dims, act_dims)) * n


def sub_spaces(world):
    """per agent, the widths of its action sub-spaces in action-vector order: [5] if movable, then [dim_c] if it speaks"""
    return [([5] if a.movable else []) + ([world.dim_c] if not a.silent else []) for a in world.agents]


def card_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = [x.strip() for x in out[0].split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001  (the number still stands; say what is missing)
        return {"error": "nvidia-smi: %s" % e}


def time_critic(args, env, mods, kw, res, e0, e1):
    """(a) the rollout with MAPPO's critic in the kernel, (b) the rollout recording observations, then the torch critic
    over the concatenated records and the final observations; device time per step of each"""
    import torch
    nn = torch.nn
    nw = env.world.native
    n, T, H, D = args.num_envs, args.steps, args.hidden, sum(nw.obs_dims)
    Act = nn.Tanh if args.tanh else nn.ReLU
    count = 1 if args.critic == "shared" else len(nw.obs_dims)
    crits = [nn.Sequential(*(([nn.LayerNorm(D)] if args.feature_norm else []) +
                             [nn.Linear(D, H), Act(), nn.LayerNorm(H), nn.Linear(H, H), Act(), nn.LayerNorm(H),
                              nn.Linear(H, 1)])).to(mods[0][0].weight.device) for _ in range(count)]
    critic = crits[0] if count == 1 else crits

    def in_kernel():
        env.rollout_policy(mods, T, critic=critic, **kw)

    def kernel_then_torch():
        obs_n, _, _, _, ex = env.rollout_policy(mods, T, record_observations=True, **kw)
        x = torch.cat(ex["observations"], -1).reshape(T * n, D)
        final = torch.cat(list(obs_n), -1)
        with torch.no_grad():
            for c in crits:
                c(x)
                c(final)

    def timed(fn):
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        e0.record()
        for _ in range(args.reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 1e3 / (args.reps * T)

    res["config"].update(torch_float32_matmul_precision=torch.get_float32_matmul_precision())
    sa, sb = timed(in_kernel), timed(kernel_then_torch)
    res["in_kernel_critic"] = {"us_per_step": 1e6 * sa, "env_steps_per_sec": n / sa}
    res["kernel_then_torch_critic"] = {"us_per_step": 1e6 * sb, "env_steps_per_sec": n / sb}
    res["speedup"] = sb / sa
    res["card"] = card_info()
    return res


def time_rcritic(args, env, mods, kw, res, e0, e1):
    """rMAPPO's recurrent critic: (a) the rollout with the critic kernel after it, (b) the rollout recording
    observations without a critic, (c) (b), then the torch critic; device time per step of each"""
    import torch
    nn = torch.nn
    nw = env.world.native
    n, T, H, D = args.num_envs, args.steps, args.hidden, sum(nw.obs_dims)
    dev = mods[0][0][-1].weight.device
    Act = nn.Tanh if args.tanh else nn.ReLU

    def make():
        base = nn.Sequential(*(([nn.LayerNorm(D)] if args.feature_norm else []) +
                               [nn.Linear(D, H), Act(), nn.LayerNorm(H), nn.Linear(H, H), Act(), nn.LayerNorm(H)]))
        return tuple(m.to(dev) for m in (base, nn.GRU(H, H), nn.LayerNorm(H), nn.Linear(H, 1)))

    crits = [make() for _ in (nw.obs_dims if args.separated else [0])]   # one per agent, or one shared
    critic = crits if args.separated else crits[0]
    h0 = torch.zeros(1, n, H, device=dev)

    def in_kernel():
        env.rollout_policy(mods, T, critic=critic, **kw)

    def recording():
        return env.rollout_policy(mods, T, record_observations=True, **kw)

    def kernel_then_torch():
        obs_n, _, _, _, ex = recording()
        x = torch.cat(ex["observations"], -1).reshape(T * n, D)
        with torch.no_grad():
            for b, gru, norm, v_out in crits:
                out, hT = gru(b(x).reshape(T, n, H), h0)
                v_out(norm(out))
                _, hb = gru(b(torch.cat(list(obs_n), -1))[None], hT)
                v_out(norm(hb[0]))

    def timed(fn):
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        e0.record()
        for _ in range(args.reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 1e3 / (args.reps * T)

    res["config"].update(torch_float32_matmul_precision=torch.get_float32_matmul_precision(),
                         cudnn_allow_tf32=torch.backends.cudnn.allow_tf32)
    sa, sr, sb = timed(in_kernel), timed(recording), timed(kernel_then_torch)
    res["in_kernel_critic"] = {"us_per_step": 1e6 * sa, "env_steps_per_sec": n / sa}
    res["rollout_recording_observations"] = {"us_per_step": 1e6 * sr, "env_steps_per_sec": n / sr}
    res["kernel_then_torch_critic"] = {"us_per_step": 1e6 * sb, "env_steps_per_sec": n / sb}
    res["critic_kernel_us_per_step"] = 1e6 * (sa - sr)
    res["speedup"] = sb / sa
    res["card"] = card_info()
    return res


def time_local_critic(args, env, mods, kw, res, e0, e1):
    """IPPO's local critics (centralized_critic=False), each critic on its agent's own observation: (a) the call with
    them in-kernel, (b) the same call without a critic (with --critic recurrent-local: recording observations, the
    critic kernel's input), (c) (b), then the same local critics in torch over the records and the final observations,
    and (d) the centralized critic in-kernel on the same program where it has a kernel; device time per step of each"""
    import torch
    from multiagent_particle_envs_b200._lib import MpeError
    nn = torch.nn
    nw = env.world.native
    n, T, H, A = args.num_envs, args.steps, args.hidden, len(nw.obs_dims)
    recurrent = args.critic == "recurrent-local"
    dev = (mods[0][0][-1] if recurrent else mods[0][0]).weight.device
    Act = nn.Tanh if args.tanh else nn.ReLU
    shared = len(set(nw.obs_dims)) == 1     # one shared critic where the agents observe alike, else one per agent

    def base(d):
        return ([nn.LayerNorm(d)] if args.feature_norm else []) + [nn.Linear(d, H), Act(), nn.LayerNorm(H),
                                                                  nn.Linear(H, H), Act(), nn.LayerNorm(H)]

    def make(d):
        if recurrent:
            return tuple(m.to(dev) for m in (nn.Sequential(*base(d)), nn.GRU(H, H), nn.LayerNorm(H), nn.Linear(H, 1)))
        return nn.Sequential(*base(d), nn.Linear(H, 1)).to(dev)

    crits = [make(nw.obs_dims[0])] * A if shared else [make(od) for od in nw.obs_dims]
    critic = crits[0] if shared else crits
    central = make(sum(nw.obs_dims))
    h0 = torch.zeros(1, n, H, device=dev)

    def in_kernel():
        env.rollout_policy(mods, T, critic=critic, centralized_critic=False, **kw)

    def actor_only():
        return env.rollout_policy(mods, T, record_observations=recurrent, **kw)

    def kernel_then_torch():
        obs_n, _, _, _, ex = env.rollout_policy(mods, T, record_observations=True, **kw)
        with torch.no_grad():
            for k, c in enumerate(crits):
                x = ex["observations"][k].reshape(T * n, -1)
                if recurrent:
                    b, gru, norm, v_out = c
                    out, hT = gru(b(x).reshape(T, n, H), h0)
                    v_out(norm(out))
                    _, hb = gru(b(obs_n[k])[None], hT)
                    v_out(norm(hb[0]))
                else:
                    c(x)
                    c(obs_n[k])

    def centralized():
        env.rollout_policy(mods, T, critic=central, **kw)

    def timed(fn):
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        e0.record()
        for _ in range(args.reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 1e3 / (args.reps * T)

    res["config"].update(torch_float32_matmul_precision=torch.get_float32_matmul_precision(),
                         local_critics="shared" if shared else "per_agent")
    sa, so, sb = timed(in_kernel), timed(actor_only), timed(kernel_then_torch)
    res["in_kernel_local_critic"] = {"us_per_step": 1e6 * sa, "env_steps_per_sec": n / sa}
    res["in_kernel_actor_only" + ("_recording_observations" if recurrent else "")] = \
        {"us_per_step": 1e6 * so, "env_steps_per_sec": n / so}
    res["kernel_then_torch_local_critic"] = {"us_per_step": 1e6 * sb, "env_steps_per_sec": n / sb}
    res["local_critic_us_per_step"] = 1e6 * (sa - so)
    res["speedup"] = sb / sa
    try:
        sc = timed(centralized)
        res["in_kernel_centralized_critic"] = {"us_per_step": 1e6 * sc, "env_steps_per_sec": n / sc}
    except MpeError as e:   # spread N=6: no centralized critic kernel
        res["in_kernel_centralized_critic"] = {"error": str(e)}
    if shared and not recurrent:   # one critic per agent, local and centralized, where they fit next to the actor
        per_agent = {"in_kernel_local_critic_per_agent": ([make(od) for od in nw.obs_dims], False),
                     "in_kernel_centralized_critic_per_agent": ([make(sum(nw.obs_dims)) for _ in range(A)], True)}
        for name, (cs, cen) in per_agent.items():
            try:
                s = timed(lambda: env.rollout_policy(mods, T, critic=cs, centralized_critic=cen, **kw))
                res[name] = {"us_per_step": 1e6 * s, "env_steps_per_sec": n / s}
            except MpeError as e:
                res[name] = {"error": str(e)}
    res["card"] = card_info()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenario", default="simple_spread")
    ap.add_argument("--scenario-kwargs", nargs="*", default=[], metavar="KEY=INT",
                    help="scenario keyword arguments, e.g. num_agents=6 or num_adversaries=6 num_good_agents=2")
    ap.add_argument("--num-envs", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=25)
    ap.add_argument("--hidden", type=int, default=64)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--layers", type=int, choices=(2, 3), default=2, help="Linear layers of the actor")
    ap.add_argument("--explore", action="store_true", help="Gumbel-softmax exploration (--layers 3)")
    ap.add_argument("--categorical", action="store_true",
                    help="one-hot arg-max actions with index and log-probability records (--layers 3)")
    ap.add_argument("--actor", choices=("maddpg", "mappo", "rmappo"), default="maddpg",
                    help="mappo: MAPPO's LayerNorm actor, rmappo: its recurrent actor (both imply --layers 3 "
                         "--categorical)")
    ap.add_argument("--tanh", action="store_true", help="MAPPO's actor with Tanh instead of ReLU")
    ap.add_argument("--feature-norm", action="store_true", help="MAPPO's actor with the input LayerNorm")
    ap.add_argument("--separated", action="store_true",
                    help="rMAPPO's separated runner: one recurrent actor (and critic) per agent (--actor rmappo)")
    ap.add_argument("--critic", choices=("shared", "separated", "recurrent", "local", "recurrent-local"),
                    help="time MAPPO's centralized critic in-kernel against the torch critic after the rollout "
                         "(shared, separated: --actor mappo; recurrent: --actor rmappo), or IPPO's local critics "
                         "(local: --actor mappo; recurrent-local: --actor rmappo)")
    args = ap.parse_args()
    if args.critic in ("shared", "separated", "local") and args.actor != "mappo":
        ap.error("--critic shared|separated|local needs --actor mappo")
    if args.critic in ("recurrent", "recurrent-local") and (args.actor != "rmappo" or args.separated):
        ap.error("--critic recurrent|recurrent-local needs --actor rmappo (recurrent-local: without --separated)")
    if args.separated and args.actor != "rmappo":
        ap.error("--separated needs --actor rmappo")
    if args.actor in ("mappo", "rmappo"):
        args.layers, args.categorical = 3, True
    elif args.tanh or args.feature_norm:
        ap.error("--tanh and --feature-norm need --actor mappo or rmappo")
    try:
        skw = {k: int(v) for k, v in (kv.split("=", 1) for kv in args.scenario_kwargs)}
    except ValueError:
        ap.error("--scenario-kwargs takes KEY=INT pairs")
    if args.explore and args.layers != 3:
        ap.error("--explore needs --layers 3")
    if args.categorical and args.layers != 3:
        ap.error("--categorical needs --layers 3")
    import torch
    import __graft_entry__ as g
    g.build(quiet=True)
    from multiagent_particle_envs_b200 import make_env
    from multiagent_particle_envs_b200.rollout import GraphedRollout
    dev = torch.device("cuda", 0)
    n, T, H = args.num_envs, args.steps, args.hidden
    env = make_env(args.scenario, num_envs=n, device=dev, **skw)
    env.reuse_buffers = True
    env.reset()
    nw = env.world.native
    torch.manual_seed(0)
    if args.layers == 2:
        mods = [torch.nn.Sequential(torch.nn.Linear(od, H), torch.nn.ReLU(), torch.nn.Linear(H, 5)).to(dev) for od in nw.obs_dims]
    else:
        mods = [torch.nn.Sequential(torch.nn.Linear(od, H), torch.nn.ReLU(), torch.nn.Linear(H, H), torch.nn.ReLU(),
                                    torch.nn.Linear(H, ad)).to(dev) for od, ad in zip(nw.obs_dims, nw.act_dims)]
    maddpg_mods = None
    if args.actor == "mappo":
        nn = torch.nn
        Act = nn.Tanh if args.tanh else nn.ReLU
        maddpg_mods = mods
        mods = [nn.Sequential(*(([nn.LayerNorm(od)] if args.feature_norm else []) +
                                [nn.Linear(od, H), Act(), nn.LayerNorm(H), nn.Linear(H, H), Act(), nn.LayerNorm(H),
                                 nn.Linear(H, ad)])).to(dev) for od, ad in zip(nw.obs_dims, nw.act_dims)]
    rnn = None
    if args.actor == "rmappo":
        nn = torch.nn
        torch.set_float32_matmul_precision("highest")
        Act = nn.Tanh if args.tanh else nn.ReLU

        def make(od, ad):
            base = nn.Sequential(*(([nn.LayerNorm(od)] if args.feature_norm else []) +
                                   [nn.Linear(od, H), Act(), nn.LayerNorm(H), nn.Linear(H, H), Act(), nn.LayerNorm(H)]))
            return tuple(m.to(dev) for m in (base, nn.GRU(H, H), nn.LayerNorm(H), nn.Linear(H, ad)))

        if args.separated:
            mods = [make(od, ad) for od, ad in zip(nw.obs_dims, nw.act_dims)]
        else:
            mods = [make(nw.obs_dims[0], nw.act_dims[0])] * len(nw.obs_dims)
        rnn = torch.zeros(len(nw.obs_dims) * n, H, device=dev)    # the graphed loop's carried h, agents stacked
    segs = sub_spaces(env.world) if args.layers == 3 else [[5]] * len(nw.obs_dims)
    res = {"config": {"scenario": args.scenario, "scenario_kwargs": skw, "n_env": n, "T": T, "hidden": H}}
    if args.layers == 3:
        res["config"].update(layers=3, explore=args.explore, categorical=args.categorical,
                             torch_float32_matmul_precision=torch.get_float32_matmul_precision())
    if args.actor in ("mappo", "rmappo"):
        res["config"].update(actor=args.actor, tanh=args.tanh, feature_norm=args.feature_norm)
    if args.separated:   # computed from the launch shape the library picks (8-warp blocks), not measured
        warps, sms = (n + 31) // 32, torch.cuda.get_device_properties(dev).multi_processor_count
        wpb = min(8, max(1, (warps + sms - 1) // sms))
        image_bytes = nw.gru_separated_workspace_bytes()
        res["config"].update(separated=True, image_bytes=image_bytes,
                             restage_bytes_per_step=(warps + wpb - 1) // wpb * image_bytes)
    kw = {"explore_seed": 1} if args.explore else {}
    if args.categorical:
        kw.update(action_mode="categorical", record_actions=True, record_log_probs=True)
    # (a) in-kernel actors
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def time_in_kernel(ms):
        for _ in range(2):
            env.rollout_policy(ms, T, **kw)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(args.reps):
            env.rollout_policy(ms, T, **kw)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 1e3 / (args.reps * T)

    if args.critic:
        res["config"].update(critic=args.critic)
        timer = {"recurrent": time_rcritic, "local": time_local_critic,
                 "recurrent-local": time_local_critic}.get(args.critic, time_critic)
        res = timer(args, env, mods, kw, res, e0, e1)
        if not args.separated:   # the separated runner's critic arms go with its rollout arms, in the same run
            print(json.dumps(res))
            return
    sec = time_in_kernel(mods)
    res["in_kernel"] = {"us_per_step": 1e6 * sec, "env_steps_per_sec": n / sec}
    if maddpg_mods is not None:   # the MADDPG categorical kernel on the same env, same sizes
        sec_m = time_in_kernel(maddpg_mods)
        res["maddpg_in_kernel"] = {"us_per_step": 1e6 * sec_m, "env_steps_per_sec": n / sec_m}
    if args.layers == 3 and rnn is None:
        flops = actor_flops_per_step(nw.obs_dims, nw.act_dims, H, n)
        res["in_kernel"].update(actor_flop_per_step=flops, actor_tflops=flops / sec / 1e12)
    # (b) torch actors + env.step in one CUDA graph
    env2 = make_env(args.scenario, num_envs=n, device=dev, **skw)
    env2.reset()

    def act(z, seg):   # one softmax per action sub-space
        if len(seg) == 1:
            return torch.softmax(z, -1)
        return torch.cat([torch.softmax(p, -1) for p in torch.split(z, seg, -1)], -1)

    def categorical(z, seg):   # one-hot of the (perturbed) arg-max per sub-space, and the log-probability
        zp = z - torch.log(-torch.log(torch.rand(z.shape, device=dev))) if args.explore else z
        hot, logp = [], 0.0
        for zs, ps in zip(torch.split(z, seg, -1), torch.split(zp, seg, -1)):
            k = ps.argmax(-1, keepdim=True)
            hot.append(torch.nn.functional.one_hot(k[:, 0], zs.shape[-1]).float())
            logp = logp + torch.log_softmax(zs, -1).gather(-1, k)[:, 0]
        logps.append(logp)
        return torch.cat(hot, -1)

    logps = []   # the graph's log-probability outputs, kept as a trainer would keep them

    def separated_policy(obs_n):   # each agent's own tuple on its own observations and its slice of rnn
        F = torch.nn.functional
        out = []
        for i, ((base, gru, norm, head), o, seg) in enumerate(zip(mods, obs_n, segs)):
            h = rnn[i * n:(i + 1) * n]
            gi = F.linear(base(o), gru.weight_ih_l0, gru.bias_ih_l0).chunk(3, 1)
            gh = F.linear(h, gru.weight_hh_l0, gru.bias_hh_l0).chunk(3, 1)
            r, z = torch.sigmoid(gi[0] + gh[0]), torch.sigmoid(gi[1] + gh[1])
            hn = (1 - z) * torch.tanh(gi[2] + r * gh[2]) + z * h
            h.copy_(hn)
            out.append(categorical(head(norm(hn)), seg))
        return out

    def recurrent_policy(obs_n):
        # torch's GRU step written out (F.linear GEMMs and pointwise kernels capture in a graph on every backend)
        F = torch.nn.functional
        if args.separated:
            return separated_policy(obs_n)
        base, gru, norm, head = mods[0]
        gi = F.linear(base(torch.cat(obs_n, 0)), gru.weight_ih_l0, gru.bias_ih_l0).chunk(3, 1)
        gh = F.linear(rnn, gru.weight_hh_l0, gru.bias_hh_l0).chunk(3, 1)
        r, z = torch.sigmoid(gi[0] + gh[0]), torch.sigmoid(gi[1] + gh[1])
        hn = (1 - z) * torch.tanh(gi[2] + r * gh[2]) + z * rnn
        rnn.copy_(hn)
        return [categorical(zz, seg) for zz, seg in zip(head(norm(hn)).split(n), segs)]

    def policy(obs_n):
        if rnn is not None:
            return recurrent_policy(obs_n)
        if args.categorical:
            return [categorical(m(o), seg) for m, o, seg in zip(mods, obs_n, segs)]
        if args.explore:   # the same Gumbel-softmax sample, noise from torch's generator
            return [act(m(o) - torch.log(-torch.log(torch.rand(o.shape[0], sum(seg), device=dev))), seg)
                    for m, o, seg in zip(mods, obs_n, segs)]
        return [act(m(o), seg) for m, o, seg in zip(mods, obs_n, segs)]

    ro = GraphedRollout(env2, policy, steps=T)
    for _ in range(2):
        ro.run()
    torch.cuda.synchronize()
    e0.record(ro.stream)
    with torch.cuda.stream(ro.stream):
        e0.record(ro.stream)
        for _ in range(args.reps):
            ro.run()
        e1.record(ro.stream)
    torch.cuda.synchronize()
    sec2 = e0.elapsed_time(e1) / 1e3 / (args.reps * T)
    res["graphed_torch"] = {"us_per_step": 1e6 * sec2, "env_steps_per_sec": n / sec2}
    res["speedup"] = sec2 / sec
    if args.layers == 3:
        res["card"] = card_info()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
