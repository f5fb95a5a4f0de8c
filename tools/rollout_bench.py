"""Acting in a simulated vectorised environment: the closed-loop slot step (act_slots) against the loop closed by hand.

The schedule is slot_decode_bench.py's: cfg3 shapes (VIMA-200M, 256 slots, Q = 32 obs tokens, Lp = 256, f16f8), 1024 episodes of
1..15 environment steps (seed 0); a slot whose episode ended takes the next episode before the next tick (admit) or is released.
Four ways to act, each over the whole schedule, alternated (a, b, c, d, a, b, c, d) in one process:

  (a) hand     step_slots -> forward_action_decoder -> mode() -> forward_action_token, eager
  (b) greedy   act_slots, eager
  (c) sampled  act_slots with an ActionSampler, eager
  (d) graph    capture_act_slots with an ActionSampler, replayed (capture time reported, not counted)

Then the same at a launch-bound size (VIMA-20M, 64 slots).  A separate torch.profiler run gives the device time of the action-head
kernel per launch in sampling mode (draw, log-prob, entropy, plus the counter's one-thread increment) next to head_select's, on the
[S, 700] logits of one step.  Weights are random (timing only).  Prints the GPU's name and power limit beside the numbers, one
JSON line per run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import vima_b200
from oracle import synth  # model shapes only


def gpu_info() -> str:
    """Name and power limit of the card torch runs on: nvidia-smi is asked by PCI bus id, since its device indices need not be
    torch's (CUDA_VISIBLE_DEVICES)."""
    p = torch.cuda.get_device_properties(torch.cuda.current_device())
    bus = f"{p.pci_domain_id:08X}:{p.pci_bus_id:02X}:{p.pci_device_id:02X}.0"
    try:
        r = subprocess.run(["nvidia-smi", "-i", bus, "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30, check=True)
        return f"{r.stdout.strip()} (PCI {bus})"
    except Exception:  # noqa: BLE001 -- the name alone is still worth printing
        return f"{p.name} (PCI {bus}), power limit not readable"


def run_size(model, S, a, info):
    pol = vima_b200.VIMAPolicy(**synth.MODEL_CFGS[model]).cuda().eval()
    E, Q, Lp = pol.embed_dim, a.n_obj, a.prompt_len
    Lmax = a.max_steps * (Q + 1)
    lengths = np.random.default_rng(a.seed).integers(1, a.max_steps + 1, size=a.episodes).tolist()
    total_steps = int(sum(lengths))
    g = torch.Generator(device="cuda").manual_seed(a.seed)
    obs_pool = [torch.randn(1, S, Q, E, device="cuda", generator=g) for _ in range(3)]
    msk = torch.rand(1, S, Q, device="cuda", generator=g) > 0.1
    msk[..., 0] = True
    prompts = torch.randn(Lp, S, E, device="cuda", generator=g)
    pmask = torch.ones(S, Lp, dtype=torch.bool, device="cuda")
    open_slots = lambda: pol.open_slots(S, max_tokens=Lmax, max_prompt_tokens=Lp)  # noqa: E731
    print(f"# {info}; model {model}, {S} slots, Q={Q}, Lp={Lp}, {a.precision}; {a.episodes} episodes of 1..{a.max_steps} steps "
          f"({total_steps} env-steps, seed {a.seed})", flush=True)

    def hand(cache, obs, state):
        x = pol.step_slots(cache, obs, msk, state.get("tok"))
        dists = pol.forward_action_decoder(x)
        state["tok"] = pol.forward_action_token({k: d.mode() for k, d in dists.items()})

    def slotted(step, cache):
        queue = list(range(len(lengths)))
        remaining = [0] * S
        ticks, pending, state = 0, list(range(S)), {}
        while True:
            take = pending[:len(queue)]
            if take:
                pol.admit(cache, take, prompts[:, :len(take)], pmask[:len(take)])
                for b in take:
                    remaining[b] = lengths[queue.pop(0)]
            idle = pending[len(take):]
            if idle:
                pol.release(cache, idle)
            if not any(remaining):
                break
            step(cache, obs_pool[ticks % 3], state)
            ticks += 1
            pending = []
            for b in range(S):
                if remaining[b]:
                    remaining[b] -= 1
                    if remaining[b] == 0:
                        pending.append(b)
        return ticks

    with torch.no_grad():
        c = open_slots()  # warm-up: modules, weight packing, kernel attributes
        pol.admit(c, list(range(S)), prompts, pmask)
        warm = vima_b200.ActionSampler(a.seed, "cuda")
        for _ in range(2):
            hand(c, obs_pool[0], {})
            pol.act_slots(c, obs_pool[0], msk)
            pol.act_slots(c, obs_pool[0], msk, sampler=warm)
        del c
        torch.cuda.synchronize()
        for rnd in range(2):
            for name in ("hand", "greedy", "sampled", "graph"):
                cache = open_slots()
                extra = {}
                if name == "hand":
                    step = hand
                elif name == "greedy":
                    step = lambda c, o, st: pol.act_slots(c, o, msk)  # noqa: E731
                elif name == "sampled":
                    sampler = vima_b200.ActionSampler(a.seed, "cuda")
                    step = lambda c, o, st: pol.act_slots(c, o, msk, sampler=sampler)  # noqa: E731
                else:
                    sampler = vima_b200.ActionSampler(a.seed, "cuda")
                    pol.admit(cache, list(range(S)), prompts, pmask)
                    t0 = time.perf_counter()
                    gs = pol.capture_act_slots(cache, obs_pool[0], msk, sampler=sampler)
                    torch.cuda.synchronize()
                    extra = {"capture_s": round(time.perf_counter() - t0, 3), "vima_kernels_per_replay": gs.kernels_per_replay}
                    pol.release(cache, list(range(S)))
                    step = lambda c, o, st: gs(o, msk)  # noqa: E731
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                ticks = slotted(step, cache)
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                r = {"model": model, "slots": S, "run": name, "round": rnd, "seconds": round(dt, 4), "ticks": ticks,
                     "env_steps_per_s": round(total_steps / dt, 1), "ms_per_tick": round(dt * 1e3 / ticks, 3)}
                r.update(extra)
                r["gpu"] = info
                print(json.dumps(r), flush=True)
                del cache
        # kernel device time: head_select vs the sampling launch on one step's logits, profiled on their own
        dims = [n for d in pol.action_decoder._decoders.values() for n in d.mlps_and_dims()[1]]
        logits = torch.randn(S, sum(dims), device="cuda")
        sampler = vima_b200.ActionSampler(a.seed, "cuda")
        from torch.profiler import ProfilerActivity, profile

        from vima_b200.nn.action import sample_heads, select_heads

        kern = {}
        reps = 200
        for name, fn in (("head_select", lambda: select_heads(logits, dims)),
                         ("head_sample", lambda: sample_heads(logits, dims, sampler=sampler, log_prob=True, entropy=True))):
            for _ in range(10):
                fn()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(reps):
                    fn()
                torch.cuda.synchronize()
            us = {}
            for ev in prof.events():
                if ev.device_type == torch.autograd.DeviceType.CUDA and ("head_kernel" in ev.name or "counter_increment" in ev.name):
                    key = "head_kernel" if "head_kernel" in ev.name else "counter_increment"
                    us[key] = us.get(key, 0.0) + ev.device_time / reps
            kern[name] = {k: round(v, 2) for k, v in us.items()}
        print(json.dumps({"model": model, "slots": S, "kernel_us_per_launch": kern, "logits": [S, sum(dims)], "gpu": info}), flush=True)
    del pol
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="200M:256,20M:64", help="model:slots pairs")
    ap.add_argument("--n-obj", type=int, default=32)
    ap.add_argument("--prompt-len", type=int, default=256)
    ap.add_argument("--max-steps", type=int, default=15)
    ap.add_argument("--episodes", type=int, default=1024)
    ap.add_argument("--precision", default="f16f8")
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("rollout_bench needs a CUDA device")
    vima_b200.set_precision(a.precision)
    torch.manual_seed(a.seed)
    info = gpu_info()
    for item in a.sizes.split(","):
        model, S = item.split(":")
        run_size(model, int(S), a, info)


if __name__ == "__main__":
    main()
