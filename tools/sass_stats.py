#!/usr/bin/env python
"""Static view of every fused-step kernel in libmpe_b200.so (no GPU needed): registers / stack from
`cuobjdump -res-usage`, instruction mix from `cuobjdump -sass`.  The counts are STATIC instructions of the whole
kernel; every entity loop is unrolled, but the runtime-selected alternatives (the partial-warp tail path with scalar
loads / stores, exact-image vs padded tile streaming) are all in the binary, so a
full warp executes roughly half of them (spread N=3: 664 executed per warp in ncu vs 1252 static).

    python tools/sass_stats.py > profiles/r1_static_resources.md

`--compare OTHER.so` instead compares this library's kernels with OTHER's, function by function: which exist in only
one of them, which have different SASS, and which changed registers or stack; it exits with 1 if anything differs.
"Different SASS" compares the instruction text (opcode, operands and the address/encoding line cuobjdump prints with
it), not the separate control-word line (stall counts, yield, barriers, operand reuse), so two builds that differ
only in scheduling control bits count as the same.

    python tools/sass_stats.py --compare /path/to/parent/libmpe_b200.so
"""
import argparse
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.environ.get("MPE_B200_LIB", os.path.join(ROOT, "multiagent_particle_envs_b200", "csrc", "libmpe_b200.so"))


def demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.split("\n")
    return dict(zip(names, out))


def resource_usage(lib):
    """{mangled name: (registers, stack bytes)} from `cuobjdump -res-usage`."""
    res = subprocess.run(["cuobjdump", "-res-usage", lib], capture_output=True, text=True, check=True).stdout
    usage = {}
    cur = None
    for ln in res.splitlines():
        m = re.match(r"\s*Function (\S+):", ln)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+)", ln)
        if m and cur:
            usage[cur] = (int(m.group(1)), int(m.group(2)))
            cur = None
    return usage


def sass_text(lib):
    """{mangled name: the function's SASS instruction lines} from `cuobjdump -sass`."""
    sass = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    funcs = {}
    cur = None
    for ln in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", ln)
        if m:
            cur = funcs.setdefault(m.group(1), [])
            continue
        if cur is not None and re.match(r"\s*/\*[0-9a-f]{4,}\*/", ln):
            cur.append(ln.strip())
    return funcs


def compare(other):
    a_sass, b_sass = sass_text(LIB), sass_text(other)
    a_use, b_use = resource_usage(LIB), resource_usage(other)
    names = demangle(sorted(set(a_sass) | set(b_sass) | set(a_use) | set(b_use)))
    print("this: %s (%d functions)\nother: %s (%d functions)" % (LIB, len(a_sass), other, len(b_sass)))
    only_a = sorted(names[k] for k in set(a_sass) - set(b_sass))
    only_b = sorted(names[k] for k in set(b_sass) - set(a_sass))
    differ = sorted(names[k] for k in set(a_sass) & set(b_sass) if a_sass[k] != b_sass[k])
    usage = sorted((names[k], b_use[k], a_use[k]) for k in set(a_use) & set(b_use) if a_use[k] != b_use[k])
    print("\nonly in this library: %d" % len(only_a))
    for nm in only_a:
        print("  " + nm)
    print("\nonly in the other library: %d" % len(only_b))
    for nm in only_b:
        print("  " + nm)
    print("\ndifferent SASS: %d of %d" % (len(differ), len(set(a_sass) & set(b_sass))))
    for nm in differ:
        print("  " + nm)
    print("\nREG / STACK changed (other -> this): %d" % len(usage))
    for nm, (rb, sb), (ra, sa) in usage:
        print("  %s: REG %d -> %d, STACK %d -> %d" % (nm, rb, ra, sb, sa))
    return 1 if only_a or only_b or differ or usage else 0


def main():
    usage = resource_usage(LIB)
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
    mix = {}
    cur = None
    for ln in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", ln)
        if m:
            cur = m.group(1)
            mix[cur] = collections.Counter()
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)(\.[A-Z0-9_.]+)?", ln)
        if m and cur:
            op = m.group(1)
            if op == "NOP":
                continue
            mix[cur]["total"] += 1
            mix[cur][op] += 1
            if op == "MUFU":
                mix[cur]["MUFU" + (m.group(2) or "")] += 1
    names = demangle(sorted(usage))
    rows = []
    for mangled, (reg, stack) in usage.items():
        nm = names[mangled]
        m = re.match(r"void mpe::mpe_kernel<mpe::(.+), 0, (false|true), (false|true)>\(", nm)
        if not m:
            continue
        label = m.group(1) + (" HOT" if m.group(2) == "true" else "") + (" 80-reg" if m.group(3) == "true" else "")
        c = mix.get(mangled, {})
        fp = sum(c[k] for k in ("FADD", "FMUL", "FFMA", "FSETP", "FSEL", "FMNMX", "FMNMX3"))
        rows.append((label, reg, stack, c["total"], fp, c["MUFU"], c["LDG"], c["LDGSTS"], c["LDS"], c["STS"], c["STG"],
                     c["BRA"] + c["BSSY"] + c["BSYNC"], c["WARPSYNC"] + c["BAR"]))
    rows.sort(key=lambda r: r[3])
    print("# Static resources of the fused-step kernels (`tools/sass_stats.py`, sm_90a, %s)\n" % os.path.basename(LIB))
    print("`__launch_bounds__(512, 1)` caps registers at 128.  No kernel spills (STACK 0).  Columns are static SASS counts of "
          "the whole kernel including the runtime-selected alternatives (partial-warp tail), NOPs excluded; `fp` = FADD+FMUL+FFMA+FSETP+FSEL+FMNMX, `branch` = BRA+BSSY+BSYNC.\n")
    print("| program | regs | stack | instr | fp | MUFU | LDG | LDGSTS | LDS | STS | STG | branch | sync |")
    print("|---|---|---|---|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        print("| " + " | ".join(str(x) for x in r) + " |")
    forms = {"mlp_rollout": "S", "mlp_episode": "E", "mlp_categorical": "C", "mlp_categorical_episode": "CE",
             "mappo": "M", "mappo_episode": "ME", "gru": "G", "gru_episode": "GE", "mappo_critic": "V",
             "mappo_critic_episode": "VE", "critic_gru": "R", "gru_separated": "GS", "gru_separated_episode": "GSE",
             "critic_gru_separated": "RS", "gru_image": "I", "mappo_local_critic": "L",
             "mappo_local_critic_episode": "LE", "critic_gru_local": "RL"}
    mlp = []
    for mangled, (reg, stack) in usage.items():
        m = re.match(r"void mpe::mpe_(?:policy_)?(mlp_rollout|mlp_episode|mlp_categorical|mlp_categorical_episode|mappo|"
                     r"mappo_episode|gru|gru_episode|mappo_critic|mappo_critic_episode|critic_gru|gru_separated|"
                     r"gru_separated_episode|critic_gru_separated|gru_image|mappo_local_critic|"
                     r"mappo_local_critic_episode|critic_gru_local)_kernel<mpe::(.+?)"
                     r"(?:, (\d+))?\s*>\(", names[mangled])
        if m:
            c = mix.get(mangled, {})
            mlp.append((m.group(2), m.group(3) or "64", forms[m.group(1)], reg, stack, c["total"], c["HMMA"], c["LDS"],
                        c["MUFU"]))
    if mlp:
        print("\n## Closed-loop rollout with the two-hidden-layer actor (TF32 mma.sync), by form: S "
              "`mpe_policy_mlp_rollout_kernel`, E its episode form `mpe_policy_mlp_episode_kernel`, C and CE the "
              "categorical forms of both, M and ME MAPPO's LayerNorm actor `mpe_policy_mappo[_episode]_kernel`, G and GE its "
              "recurrent actor `mpe_policy_gru[_episode]_kernel`, V and VE its LayerNorm actor with the centralized critic "
              "`mpe_policy_mappo_critic[_episode]_kernel`, R rMAPPO's recurrent critic `mpe_critic_gru_kernel`, GS and "
              "GSE per-agent recurrent actors `mpe_policy_gru_separated[_episode]_kernel`, RS per-agent recurrent critics "
              "`mpe_critic_gru_separated_kernel`, I their fragment images `mpe_gru_image_kernel`, L and LE the LayerNorm "
              "actor with IPPO's local critics `mpe_policy_mappo_local_critic[_episode]_kernel`, RL rIPPO's recurrent "
              "local critic `mpe_critic_gru_local_kernel` (all H = 64)\n")
        print("| program | H | form | regs | stack | instr | HMMA | LDS | MUFU |")
        print("|---|---|---|---|---|---|---|---|---|")
        for r in sorted(mlp):
            print("| " + " | ".join(str(x) for x in r) + " |")
    gae = sorted((names[k].split("(")[0], reg, stack, mix.get(k, {}).get("total", 0)) for k, (reg, stack) in usage.items()
                 if re.match(r"(void )?mpe::mpe_gae_", names[k]))
    if gae:
        print("\n## GAE and returns (`mpe_gae`): the scan without and with the fp64 sums, and the normalisation\n")
        print("| kernel | regs | stack | instr |")
        print("|---|---|---|---|")
        for r in gae:
            print("| `%s` | %d | %d | %d |" % r)
    other = [(names[k], v) for k, v in usage.items() if "mpe_kernel" not in names[k] or ", 0, " not in names[k]]
    spills = [n for n, (r, s) in other if s]
    print("\nOther kernels with a non-zero stack frame: %s" % (", ".join("`%s`" % s for s in spills) or "none"))


if __name__ == "__main__":
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--compare", metavar="OTHER.so", help="compare every kernel's SASS and REG / STACK with OTHER.so")
    args = ap.parse_args()
    sys.exit(compare(args.compare) if args.compare else main())
