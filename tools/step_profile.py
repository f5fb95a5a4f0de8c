"""Where the device time of one benchmark step goes, per kernel.

    python tools/step_profile.py [--workload cfg3] [--precision f16f8] [--steps 3] [--warmup 3] [--instances 8]

Runs the bench.py policy step eagerly (kernel by kernel, not from the CUDA graph) under torch.profiler with CUDA activities
and prints, per kernel name (template arguments dropped), the device time per step and its share of the summed kernel time
of the step; then the most expensive template instantiations.  Profile in a run of its own: the profiler slows the host, so
the event-timed step printed here is not the benchmark's number.
"""
import argparse
import collections
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import bench  # noqa: E402


def base_name(name: str) -> str:
    name = re.sub(r"^void\s+", "", name).replace("(anonymous namespace)::", "")
    depth, out = 0, []
    for ch in name:  # drop template arguments (they nest) and the parameter list
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0:
            break
        elif depth == 0:
            out.append(ch)
    return "".join(out).strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg3", choices=["cfg3", "cfg2", "cfg3x", "cfg5"])
    ap.add_argument("--precision", default="f16f8")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--instances", type=int, default=8, help="template instantiations listed after the per-name table")
    args = ap.parse_args()

    import vima_b200
    from vima_b200.utils import DataDict

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    vima_b200.set_precision(args.precision)
    wl = bench.Workload(args.workload)
    with torch.no_grad():
        policy = bench.build_our_policy(wl, dev)
        prompt_tokens, prompt_masks, _ = bench.encode_prompt(policy, wl, dev)
        inputs = bench.host_inputs(wl)
        step = bench.Stepper(policy, DataDict, wl, dev, inputs, prompt_tokens, prompt_masks)
        obs = bench.to_dev(bench.pin(inputs["new"]), dev)
        for _ in range(args.warmup):
            step(obs)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            e0.record()
            for _ in range(args.steps):
                step(obs)
            e1.record()
            torch.cuda.synchronize()
        step_ms = e0.elapsed_time(e1) / args.steps

    per_name = collections.defaultdict(lambda: [0.0, 0])
    per_inst = collections.defaultdict(lambda: [0.0, 0])
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        us = ev.time_range.elapsed_us()
        for table, key in ((per_name, base_name(ev.name)), (per_inst, ev.name)):
            table[key][0] += us
            table[key][1] += 1
    busy_ms = sum(v[0] for v in per_name.values()) / 1e3 / args.steps
    props = torch.cuda.get_device_properties(dev)
    print(f"{args.workload} {args.precision} on {props.name}: eager step {step_ms:.3f} ms (event-timed, profiled), "
          f"device kernel time {busy_ms:.3f} ms/step over {args.steps} steps")
    print(f"{'kernel':60s} {'ms/step':>9s} {'share':>7s} {'launches/step':>14s}")
    for key, (us, n) in sorted(per_name.items(), key=lambda kv: -kv[1][0]):
        ms = us / 1e3 / args.steps
        print(f"{key[:60]:60s} {ms:9.3f} {ms / busy_ms:7.1%} {n / args.steps:14.1f}")
    print(f"\ntop {args.instances} instantiations")
    for key, (us, n) in sorted(per_inst.items(), key=lambda kv: -kv[1][0])[:args.instances]:
        ms = us / 1e3 / args.steps
        print(f"{ms:9.3f} ms/step {ms / busy_ms:7.1%}  x{n / args.steps:.0f}  {key}")


if __name__ == "__main__":
    main()
