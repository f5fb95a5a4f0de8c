"""Slot decode vs lockstep decode in a simulated vectorised environment (cfg3 shapes: 200M, 256 slots, Q = 32 obs tokens, Lp = 256).

With --policy gato | gpt | flamingo the same simulation runs on a baseline policy (e.g. `--policy gato --model gato_200M`: cfg5
shapes, 22 layers, Q = 16 tokens per observation).  The decoder-only baselines hold prompt + separator in the cache, so a slot has
Lp + 1 + --max-steps * (Q + 1) columns (512 at cfg5), and a fourth run is added in front:

  reforward  forward over the whole growing history every step, as the reference's env loop does (episodes in batches of --slots)

Episode lengths are drawn from a seeded uniform distribution over 1..--max-steps environment steps (15 * 33 tokens fit the 512
positions).  Every episode runs to its end in each of three runs, and each run reports completed env-steps/s and episodes/s:

  lockstep  start_decode / forward_step: episodes go in batches of --slots and a batch runs until its longest episode ends
  eager     open_slots / step_slots: a slot whose episode ended takes the next episode before the next tick (admit), or is released
  graph     the same schedule with the step replayed from one CUDA graph (capture time reported, not counted)

Longer episodes need more decoder positions: `--policy gato --model gato_200M --n-positions 1024 --max-steps 45` gives each slot
257 + 45 * 17 = 1022 columns.  The header line prints the unpaged K/V size (n_layer * S * Lmax * 2E * 4 bytes), the slot runs'
page pool (--kv-pool-tokens, default S * Lmax rounded up to 64-token pages per slot) and the schedule's peak and mean page count;
each slot run reports the peak pages it used and torch.cuda.max_memory_allocated.

Admission (the prompt key/value GEMMs of the new episodes) is included in the slot runs' totals and also reported on its own
(CUDA events).  Weights are random (timing only).  Prints the GPU's name and power limit beside the numbers, one JSON line per run.
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
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        line = r.stdout.strip().splitlines()[torch.cuda.current_device()]
        return line
    except Exception:  # noqa: BLE001 -- the name alone is still worth printing
        return f"{torch.cuda.get_device_name()}, power limit not readable"


def pages_per_tick(lengths, S: int, Q: int, prefix: int, page: int = 64) -> list:
    """K/V pages the active slots own at each tick of the slot runs' schedule (a slot whose episode ended takes the next one before
    the next tick): a slot at cache length len owns the pages of its columns [0, len + Q + 1) once the tick's step has reserved
    them.  A new episode starts at len = prefix (prompt + separator of the decoder-only baselines, 0 otherwise); its first step adds
    Q columns (the dummy row is overwritten), every later one Q + 1.  Host arithmetic only."""
    queue = list(lengths)
    remaining, length = [0] * S, [0] * S
    out = []
    while True:
        for b in range(S):
            if not remaining[b] and queue:
                remaining[b], length[b] = queue.pop(0), prefix
        active = [b for b in range(S) if remaining[b]]
        if not active:
            return out
        out.append(sum(-(-(length[b] + Q + 1) // page) for b in active))
        for b in active:
            length[b] += Q + (length[b] != prefix)
            remaining[b] -= 1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--policy", default="vima", choices=["vima", "gato", "gpt", "flamingo"])
    ap.add_argument("--model", default=None, help="synth config name (default: 200M for vima, gato_200M for gato / gpt, flamingo_tiny)")
    ap.add_argument("--slots", type=int, default=256)
    ap.add_argument("--n-obj", type=int, default=32)
    ap.add_argument("--prompt-len", type=int, default=256)
    ap.add_argument("--max-steps", type=int, default=15)
    ap.add_argument("--n-positions", type=int, default=None,
                    help="decoder positions (default: the policy's 512); gato / gpt: the constructor's n_positions, vima: XAttnGPT rebuilt")
    ap.add_argument("--episodes", type=int, default=1024)
    ap.add_argument("--precision", default="f16f8")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--kv-pool-tokens", type=int, default=None,
                    help="K/V page pool of the slot runs, in tokens (default: slots * Lmax rounded up to pages; 'peak' sizes use the "
                         "schedule's peak page count printed in the header)")
    ap.add_argument("--runs", default=None, help="default: lockstep,eager,graph (vima); reforward,lockstep,eager,graph (baselines)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("slot_decode_bench needs a CUDA device")
    vima_b200.set_precision(a.precision)
    torch.manual_seed(a.seed)
    vima = a.policy == "vima"
    npos = {} if a.n_positions is None else {"n_positions": a.n_positions}
    if vima:
        cfg = synth.MODEL_CFGS[a.model or "200M"]
        pol = vima_b200.VIMAPolicy(**cfg)
        if npos:
            from vima_b200 import nn as vnn

            pol.xattn_gpt = vnn.XAttnGPT(cfg["embed_dim"], n_layer=cfg["xf_n_layers"], n_head=cfg["sattn_n_heads"], dropout=0.1,
                                         xattn_n_head=cfg["xattn_n_heads"], xattn_ff_expanding=4, xattn_n_positions=256, use_geglu=True,
                                         **npos)
        pol = pol.cuda().eval()
    elif a.policy == "flamingo":
        if npos:
            raise SystemExit("--n-positions applies to --policy vima, gato and gpt")
        pol = vima_b200.VIMAFlamingoPolicy(**synth.FLAMINGO_CFGS[a.model or "flamingo_tiny"]).cuda().eval()
    else:
        cls = vima_b200.VIMAGatoPolicy if a.policy == "gato" else vima_b200.VIMAGPTPolicy
        pol = cls(**synth.GATO_CFGS[a.model or "gato_200M"], **npos).cuda().eval()
    E, S, Lp = pol.embed_dim, a.slots, a.prompt_len
    Q = a.n_obj if vima else pol._obj_xf_num_queries
    prefix = Lp + 1 if a.policy in ("gato", "gpt") else 0  # the decoder-only caches hold prompt + separator
    Lmax = prefix + a.max_steps * (Q + 1)
    runs = (a.runs or ("lockstep,eager,graph" if vima else "reforward,lockstep,eager,graph")).split(",")
    lengths = np.random.default_rng(a.seed).integers(1, a.max_steps + 1, size=a.episodes).tolist()
    total_steps = int(sum(lengths))
    g = torch.Generator(device="cuda").manual_seed(a.seed)
    obs_shape = (1, S, E) if a.policy == "gpt" else (1, S, Q, E)
    obs_pool = [torch.randn(*obs_shape, device="cuda", generator=g) for _ in range(3)]
    msk = torch.rand(1, S, Q, device="cuda", generator=g) > 0.1
    msk[..., 0] = True
    act = torch.randn(1, S, E, device="cuda", generator=g)
    prompts = torch.randn(Lp, S, E, device="cuda", generator=g)
    pmask = torch.ones(S, Lp, dtype=torch.bool, device="cuda")
    info = gpu_info()
    name = "" if vima else f"policy {a.policy}, "
    n_layer = pol.xattn_gpt.n_layer if hasattr(pol, "xattn_gpt") else pol.transformer.n_layer
    kv_bytes = n_layer * S * Lmax * 2 * E * 4  # per layer [S*Lmax, 2E] K|V as (hi, lo) 16-bit pairs
    page_ld = -(-Lmax // 64)
    pool_pages = S * page_ld if a.kv_pool_tokens is None else -(-a.kv_pool_tokens // 64)
    pool_bytes = n_layer * (pool_pages + 1) * 64 * 2 * E * 4  # the slot runs' page pool, zero page included
    sched = pages_per_tick(lengths, S, Q, prefix)
    # cross-attention policies: the projected prompt K/V in their own pool (default size: a full prompt in every slot)
    prompt_pages = S * -(-Lp // 64)
    prompt_pool = (f", prompt pool {prompt_pages} pages = {n_layer * (prompt_pages + 1) * 64 * 2 * E * 4 / 1e9:.2f} GB"
                   if a.policy in ("vima", "flamingo") else "")
    print(f"# {info}; {name}model {a.model or '200M'}, {S} slots, Q={Q}, Lp={Lp}, {a.precision}; {a.episodes} episodes of 1..{a.max_steps} steps "
          f"({total_steps} env-steps, seed {a.seed}); {Lmax} cache columns per slot, K/V cache {kv_bytes / 1e9:.2f} GB unpaged (S*Lmax), "
          f"page pool {pool_pages} pages = {pool_bytes / 1e9:.2f} GB{prompt_pool}; the schedule's peak {max(sched)} pages, mean "
          f"{sum(sched) / len(sched):.0f}")

    if vima:
        forward_step, step_slots = pol.forward_step, pol.step_slots
        open_slots = lambda: pol.open_slots(S, max_tokens=Lmax, max_prompt_tokens=Lp, kv_pool_tokens=a.kv_pool_tokens)  # noqa: E731
        capture = pol.capture_step_slots
        replay = lambda gs, o, m, x: gs(o, m, x)  # noqa: E731
    else:
        forward_step = lambda c, o, m, x: pol.forward_step(c, o, x)  # noqa: E731
        step_slots = lambda c, o, m, x: pol.step_slots(c, o, x)  # noqa: E731
        open_slots = lambda: pol.open_slots(S, max_tokens=Lmax, kv_pool_tokens=a.kv_pool_tokens)  # noqa: E731
        capture = lambda c, o, m, x: pol.capture_step_slots(c, o, x)  # noqa: E731
        replay = lambda gs, o, m, x: gs(o, x)  # noqa: E731

    def reforward():
        """forward over the whole history at every step (episodes in batches of S, a batch runs until its longest episode ends)."""
        obs_hist = torch.cat([obs_pool[t % 3] for t in range(a.max_steps)], 0)
        msk_hist = msk.expand(a.max_steps, *msk.shape[1:])
        act_hist = act.expand(a.max_steps, *act.shape[1:])
        ticks = 0
        for i in range(0, len(lengths), S):
            batch = lengths[i:i + S]
            n = len(batch)
            for t in range(max(batch)):
                at = None if t == 0 else act_hist[:t, :n]
                if vima:
                    pol.forward(obs_hist[:t + 1, :n], msk_hist[:t + 1, :n], at, prompts[:, :n], pmask[:n])
                else:
                    pol.forward(obs_hist[:t + 1, :n], at, prompts[:, :n], pmask[:n])
                ticks += 1
        return ticks, 0.0, None

    def lockstep():
        ticks = 0
        for i in range(0, len(lengths), S):
            batch = lengths[i:i + S]
            n = len(batch)
            cache = pol.start_decode(prompts[:, :n], pmask[:n], max_tokens=Lmax)
            for t in range(max(batch)):
                forward_step(cache, obs_pool[t % 3][:, :n], msk[:, :n], None if t == 0 else act[:, :n])
                ticks += 1
        return ticks, 0.0, None

    def slotted(step, cache):
        """Runs every episode through `cache`; returns (ticks, admission ms, peak K/V pages in use)."""
        queue = list(range(len(lengths)))
        remaining = [0] * S
        adm_ms, ticks, peak = [], 0, 0
        pending = list(range(S))  # free slots waiting for an episode
        while True:
            take = pending[:len(queue)]
            if take:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                pol.admit(cache, take, prompts[:, :len(take)], pmask[:len(take)])
                e1.record()
                adm_ms.append((e0, e1))
                for b in take:
                    remaining[b] = lengths[queue.pop(0)]
            idle = pending[len(take):]
            if idle:
                pol.release(cache, idle)
            if not any(remaining):
                break
            step(cache, obs_pool[ticks % 3], msk, act)
            peak = max(peak, cache.kv_pages_total - cache.kv_pages_free)
            ticks += 1
            pending = []
            for b in range(S):
                if remaining[b]:
                    remaining[b] -= 1
                    if remaining[b] == 0:
                        pending.append(b)
        torch.cuda.synchronize()
        return ticks, sum(e0.elapsed_time(e1) for e0, e1 in adm_ms), peak

    results = []
    with torch.no_grad():
        # warm-up: modules, weight packing, kernel attributes
        c = open_slots()
        n_w = min(S, c.kv_pages_total // -(-(prefix + 2 * Q + 2) // 64))  # slots the pool holds for two steps
        pol.admit(c, list(range(n_w)), prompts[:, :n_w], pmask[:n_w])
        for _ in range(2):
            step_slots(c, obs_pool[0], msk, act)
        del c
        if "lockstep" in runs:  # an unpaged [S*Lmax] cache
            cd = pol.start_decode(prompts, pmask, max_tokens=Lmax)
            for t in range(2):
                forward_step(cd, obs_pool[0], msk, None if t == 0 else act)
            del cd
        torch.cuda.synchronize()
        for name in runs:
            cache = fn = None  # the previous run's cache goes before the next one is opened
            extra = {}
            if name == "reforward":
                fn = reforward
            elif name == "lockstep":
                fn = lockstep
            elif name == "eager":
                cache = open_slots()
                fn = lambda: slotted(step_slots, cache)  # noqa: E731
            elif name == "graph":
                cache = open_slots()
                n_cap = min(S, cache.kv_pages_total // -(-(prefix + Q + 1) // 64))  # a small pool cannot hold every slot's first step
                pol.admit(cache, list(range(n_cap)), prompts[:, :n_cap], pmask[:n_cap])
                t0 = time.perf_counter()
                gs = capture(cache, obs_pool[0], msk, act)
                torch.cuda.synchronize()
                extra = {"capture_s": round(time.perf_counter() - t0, 3), "vima_kernels_per_replay": gs.kernels_per_replay}
                pol.release(cache, list(range(n_cap)))
                fn = lambda: slotted(lambda c, o, m, x: replay(gs, o, m, x), cache)  # noqa: E731
            else:
                raise SystemExit(f"unknown run {name}")
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            torch.cuda.reset_peak_memory_stats()
            ticks, adm, peak = fn()
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            r = {"run": name, "seconds": round(dt, 4), "ticks": ticks, "env_steps_per_s": round(total_steps / dt, 1),
                 "episodes_per_s": round(len(lengths) / dt, 2), "ms_per_tick": round(dt * 1e3 / ticks, 3)}
            if name not in ("lockstep", "reforward"):
                r["admission_ms_total"] = round(adm, 2)
                r["admission_ms_per_episode"] = round(adm / len(lengths), 4)
            r.update(extra)
            r["gpu"] = info
            r["cache_columns"] = Lmax
            r["kv_cache_bytes"] = kv_bytes
            r["max_memory_allocated"] = torch.cuda.max_memory_allocated()
            if peak is not None:
                r["kv_pool_pages"] = pool_pages
                r["kv_pool_bytes"] = pool_bytes
                r["peak_pages_used"] = peak
            results.append(r)
            print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
