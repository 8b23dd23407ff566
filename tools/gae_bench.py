#!/usr/bin/env python
"""MAPPO's GAE and returns over a finished [T, n, N] buffer, four ways, timed alternately in one run with CUDA events:
  "kernel":      env.compute_gae (mpe_gae: one scan kernel; in the normalised cases the fp64 sums, then the
                 normalisation), called eagerly from Python: the argument checks and the ctypes call are in its time;
  "kernel_graph": the same call captured in one CUDA graph: the device time of mpe_gae alone;
  "torch_loop":  MAPPO's SharedReplayBuffer.compute_returns (use_gae) transcribed in torch on the GPU -- a Python loop
                 over reversed(range(T)) of elementwise ops on [n, N] tensors, with ValueNorm's denormalisation of
                 both values in every step -- then the PPO update's advantages returns - denormalize(value_preds) and,
                 in the normalised cases, (A - mean) / (std + 1e-5) with the population std;
  "torch_graph": the same loop captured in one CUDA graph, so that launch overhead is not all that is compared.
Every case is run plain (no ValueNorm, raw advantages) and with a shared ValueNorm and advantage normalisation.
Reported per case: device time per call of each arm (median over the windows), the algorithmic bytes (16 per entry --
rewards and values read, returns and advantages written -- plus the final values, plus 8 per entry to normalise) and
their fraction of 3.35 TB/s (H100 SXM HBM3 data sheet) at kernel_graph's time, the largest |returns| difference between
the kernel and the torch loop, and the card's name and power limit read in the same run.

    python tools/gae_bench.py [--windows 7] [--calls 20]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_BYTES_PER_S = 3.35e12
GAMMA, LAM = 0.99, 0.95
# (label, worlds, T, episode_length): MAPPO's MPE buffer (T = 25), the README's categorical example (T = 128), the
# episode form (E = 8 episodes of 25), and a small batch whose columns are serial chains of T steps
CASES = [("spread3_65536_T25", 65536, 25, None), ("spread3_65536_T128", 65536, 128, None),
         ("spread3_65536_E8xL25", 65536, 200, 25), ("spread3_1024_T25", 1024, 25, None)]


def card_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = [x.strip() for x in out[0].split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001  (the number still stands; say what is missing)
        return {"error": "nvidia-smi: %s" % e}


def torch_compute_returns(rew, val, final, L, value_norm, normalize):
    """MAPPO's compute_returns (use_gae, masks from the episode layout, every episode end a truncation bootstrapped
    with its final value) and the PPO update's advantages, in torch"""
    import torch
    T = rew.shape[0]
    if value_norm is not None:
        mean, std = value_norm[0], value_norm[1]
        denorm = lambda v: v * std + mean   # noqa: E731
    else:
        denorm = lambda v: v                # noqa: E731
    ret = torch.empty_like(rew)
    gae = torch.zeros_like(rew[0])
    for step in reversed(range(T)):
        if (step + 1) % L == 0:             # last step of episode (step + 1) // L - 1: masks[step + 1] = 0 for gae
            delta = rew[step] + GAMMA * denorm(final[(step + 1) // L - 1]) - denorm(val[step])
            gae = delta
        else:
            delta = rew[step] + GAMMA * denorm(val[step + 1]) - denorm(val[step])
            gae = delta + GAMMA * LAM * gae
        ret[step] = gae + denorm(val[step])
    adv = ret - denorm(val)
    if normalize:
        adv = (adv - adv.mean()) / (adv.std(unbiased=False) + 1e-5)
    return ret, adv


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--windows", type=int, default=7, help="timed windows per arm, alternated")
    ap.add_argument("--calls", type=int, default=20, help="calls per window")
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("gae_bench needs a CUDA device")
    from multiagent_particle_envs_b200 import make_env
    print(json.dumps({"card": card_info(), "device": torch.cuda.get_device_name(0)}))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for label, N, T, L in CASES:
        env = make_env("simple_spread", num_envs=N)
        n = env.n
        E = 1 if L is None else T // L
        g = torch.Generator(device="cuda").manual_seed(0)
        rew = torch.randn(T, n, N, device="cuda", generator=g).mul_(0.5).sub_(1.0)
        val = torch.randn(T, n, N, device="cuda", generator=g)
        final = torch.randn(E, n, N, device="cuda", generator=g)
        vn_t = torch.tensor([-10.0, 4.0], device="cuda")
        for normed in (False, True):
            vn = vn_t if normed else None
            fin = final[0] if L is None else final
            arms = {"kernel": lambda: env.compute_gae(rew, val, fin, gamma=GAMMA, gae_lambda=LAM, episode_length=L,
                                                      value_norm=vn, normalize_advantages=normed),
                    "torch_loop": lambda: torch_compute_returns(rew, val, final, L or T, vn, normed)}
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                arms["kernel"]()
                arms["torch_loop"]()
                kgraph, graph = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
                with torch.cuda.graph(kgraph, stream=side):
                    arms["kernel"]()
                with torch.cuda.graph(graph, stream=side):
                    graphed_out = arms["torch_loop"]()
            torch.cuda.current_stream().wait_stream(side)
            arms = {"kernel": arms["kernel"], "kernel_graph": kgraph.replay, "torch_loop": arms["torch_loop"],
                    "torch_graph": graph.replay}
            for f in arms.values():
                for _ in range(args.warmup):
                    f()
            times = {k: [] for k in arms}
            for _ in range(args.windows):
                for k, f in arms.items():
                    e0.record()
                    for _ in range(args.calls):
                        f()
                    e1.record()
                    e1.synchronize()
                    times[k].append(e0.elapsed_time(e1) * 1e3 / args.calls)
            us = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
            k_ret, _, _ = arms["kernel"]()
            t_ret, _ = arms["torch_loop"]()
            graph.replay()
            torch.cuda.synchronize()
            entries = T * n * N
            nbytes = 16 * entries + 4 * E * n * N + (8 * entries if normed else 0)
            print(json.dumps({
                "case": label, "worlds": N, "agents": n, "T": T, "episode_length": L,
                "value_norm_and_normalize": normed, "us_per_call": {k: round(v, 2) for k, v in us.items()},
                "spread_us": {k: [round(min(v), 2), round(max(v), 2)] for k, v in times.items()},
                "bytes": nbytes,
                "kernel_graph_fraction_of_3.35TBps": round(nbytes / (us["kernel_graph"] * 1e-6) / PEAK_BYTES_PER_S, 3),
                "torch_loop_over_kernel": round(us["torch_loop"] / us["kernel"], 2),
                "torch_graph_over_kernel_graph": round(us["torch_graph"] / us["kernel_graph"], 2),
                "max_abs_ret_diff_vs_torch": float((k_ret - t_ret).abs().max()),
                "max_abs_ret_diff_graph_vs_torch": float((graphed_out[0] - t_ret).abs().max())}))
            del graph, kgraph, graphed_out
        del env, rew, val, final
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
