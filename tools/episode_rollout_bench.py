#!/usr/bin/env python
"""MADDPG experience collection, many episodes per call: the Python loop a trainer writes around one-episode calls,

    for e in range(E):
        env.rollout_policy(actors, L, <records>, explore_seed=s)
        env.reset()

against ONE call env.rollout_policy(actors, E * L, <records>, explore_seed=s, episode_length=L), which resets every world
inside the kernel between episodes.  Both explore (MADDPG collects with the Gumbel-softmax sample).  For each
(program, H, records on / off, E) the device time per env step of the batch (host clock around a synchronised window,
after a warm-up of the same shapes), the host time of one rollout_policy call on its own (the call returns before the
kernel ends, so this is the Python, weight and pointer preparation and the launch), and the card's name, power limit and
max SM clock read in the same run.  Records on = actions, per-step rewards and observations (what a replay buffer
stores); a configuration whose records would not fit --record-budget-gb is reported as skipped."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

# (label, scenario, scenario kwargs, H): the headline world, the smallest program, the largest one, and H = 32
CONFIGS = [
    ("spread N=3", "simple_spread", {}, 64),
    ("speaker_listener", "simple_speaker_listener", {}, 64),
    ("tag 6+2", "simple_tag", {"num_adversaries": 6, "num_good_agents": 2, "num_landmarks": 3}, 64),
    ("spread N=3", "simple_spread", {}, 32),
]


def record_bytes(nw, T, E):
    per_step = sum(nw.obs_dims) + sum(nw.act_dims) + nw.n_agents
    return 4 * nw.n_env * (T * per_step + E * sum(nw.obs_dims))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--num-envs", type=int, default=65536)
    ap.add_argument("--episode-length", type=int, default=25)
    ap.add_argument("--episodes", type=int, nargs="*", default=[1, 10, 40])
    ap.add_argument("--min-steps", type=int, default=2000, help="env steps per timed window")
    ap.add_argument("--rounds", type=int, default=2, help="timed windows per mode, alternating loop and episode call")
    ap.add_argument("--record-budget-gb", type=float, default=32.0)
    args = ap.parse_args()
    import torch
    import __graft_entry__ as g
    g.build(quiet=True)
    from multiagent_particle_envs_b200 import make_env
    from policy_rollout_bench import card_info
    dev = torch.device("cuda", 0)
    n, L = args.num_envs, args.episode_length
    rows = []
    for label, scenario, skw, H in CONFIGS:
        env = make_env(scenario, num_envs=n, device=dev, **skw)
        env.reset()
        nw = env.world.native
        torch.manual_seed(0)
        mods = [torch.nn.Sequential(torch.nn.Linear(od, H), torch.nn.ReLU(), torch.nn.Linear(H, H), torch.nn.ReLU(),
                                    torch.nn.Linear(H, ad)).to(dev) for od, ad in zip(nw.obs_dims, nw.act_dims)]
        for records in (True, False):
            rec = dict(record_actions=records, per_step_rewards=records, record_observations=records)
            for E in args.episodes:
                row = {"program": label, "H": H, "records": records, "E": E, "L": L, "n_env": n}
                need = record_bytes(nw, E * L, E) if records else 0
                if need > args.record_budget_gb * 2 ** 30:
                    row["skipped"] = "records need %.1f GB" % (need / 2 ** 30)
                    rows.append(row)
                    print(json.dumps(row), flush=True)
                    continue
                reps = max(1, -(-args.min_steps // (E * L)))
                host = {"loop": [], "episodes": []}

                def loop():
                    for _ in range(E):
                        t0 = time.perf_counter()
                        env.rollout_policy(mods, L, explore_seed=1, **rec)
                        host["loop"].append(time.perf_counter() - t0)
                        env.reset()

                def episodes():
                    t0 = time.perf_counter()
                    env.rollout_policy(mods, E * L, explore_seed=1, episode_length=L, **rec)
                    host["episodes"].append(time.perf_counter() - t0)

                best = {}
                for fn in (loop, episodes):             # warm-up: modules, allocator, every shape of the window
                    fn()
                torch.cuda.synchronize()
                for key in host:
                    host[key].clear()
                for _ in range(args.rounds):
                    for key, fn in (("loop", loop), ("episodes", episodes)):
                        torch.cuda.synchronize()
                        t0 = time.perf_counter()
                        for _ in range(reps):
                            fn()
                        torch.cuda.synchronize()
                        us = 1e6 * (time.perf_counter() - t0) / (reps * E * L)
                        best.setdefault(key, []).append(us)
                row.update({"loop_us_per_step": min(best["loop"]), "episodes_us_per_step": min(best["episodes"]),
                            "loop_us_per_step_all": best["loop"], "episodes_us_per_step_all": best["episodes"],
                            "speedup": min(best["loop"]) / min(best["episodes"]),
                            "host_us_per_call_loop": 1e6 * sum(host["loop"]) / len(host["loop"]),
                            "host_us_per_call_episodes": 1e6 * sum(host["episodes"]) / len(host["episodes"])})
                rows.append(row)
                print(json.dumps(row), flush=True)
                torch.cuda.empty_cache()
        del env
        torch.cuda.empty_cache()
    card = card_info()
    print(json.dumps({"card": card}))
    print("\n| program | H | records | E | loop µs/step | episode call µs/step | speed-up | host µs per call (loop / episode) |")
    print("|---|---|---|---|---|---|---|---|")
    for r in rows:
        if "skipped" in r:
            print("| %s | %d | %s | %d | skipped: %s | | | |" % (r["program"], r["H"], "on" if r["records"] else "off", r["E"],
                                                            r["skipped"]))
            continue
        print("| %s | %d | %s | %d | %.1f | %.1f | %.2fx | %.0f / %.0f |" % (
            r["program"], r["H"], "on" if r["records"] else "off", r["E"], r["loop_us_per_step"],
            r["episodes_us_per_step"], r["speedup"], r["host_us_per_call_loop"], r["host_us_per_call_episodes"]))


if __name__ == "__main__":
    main()
