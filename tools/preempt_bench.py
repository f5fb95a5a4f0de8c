"""Preemption by swapping on an overcommitted K/V pool: two drivers of the same episode schedule, alternated in one process.

The schedule is slot_decode_bench.py's: --episodes episodes of 1..--max-steps environment steps (seeded), --slots slots, cfg3 shapes
by default (VIMA-200M, Q = 32 obs tokens, Lp = 256, f16f8); `--policy gato` runs cfg5 (VIMA-Gato-200M, prompt and separator in
the history cache).  Every step is a greedy act_slots.  The history pool holds --kv-pool-tokens tokens, by default half the
schedule's peak page count, so it cannot hold every episode at its longest:

  reserve   admit an episode only when the pool has room for its worst case (--max-steps steps) on top of what the running
            episodes may still take: never refused, never preempted, but fewer episodes run at once
  swap      admit when the episode's prefix and first step fit; before each tick, while the step needs more pages than are free, swap out the
            most recently admitted active episode (policy.swap_out, to pinned host memory); swapped episodes are resumed
            (policy.swap_in), oldest first, before any new episode is admitted

Each run reports env-steps/s and episodes/s, ticks, preemptions, bytes swapped each way, the swap-out and swap-in rates (bytes over
the CUDA-event time of the swap calls), the peak pinned host bytes held by parked episodes and torch.cuda.max_memory_allocated.
An episode's k-th step takes the same inputs in both runs, so with --check the tool asserts that every episode's per-step actions
in `swap` equal those in `reserve`.  Weights are random (timing only).  Prints the GPU's name and power limit beside the numbers,
one JSON line per run.
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np
import torch

import vima_b200
from oracle import synth  # model shapes only
from slot_decode_bench import gpu_info, pages_per_tick


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--policy", default="vima", choices=["vima", "gato"])
    ap.add_argument("--model", default=None, help="synth config name (default: 200M for vima, gato_200M for gato)")
    ap.add_argument("--slots", type=int, default=256)
    ap.add_argument("--n-obj", type=int, default=32)
    ap.add_argument("--prompt-len", type=int, default=256)
    ap.add_argument("--max-steps", type=int, default=15)
    ap.add_argument("--episodes", type=int, default=1024)
    ap.add_argument("--precision", default="f16f8")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--kv-pool-tokens", type=int, default=None, help="history pool in tokens (default: half the schedule's peak pages)")
    ap.add_argument("--rounds", type=int, default=2, help="each round runs reserve then swap")
    ap.add_argument("--check", action="store_true", help="assert that both drivers take the same actions in every episode")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("preempt_bench needs a CUDA device")
    vima_b200.set_precision(a.precision)
    torch.manual_seed(a.seed)
    vima = a.policy == "vima"
    if vima:
        pol = vima_b200.VIMAPolicy(**synth.MODEL_CFGS[a.model or "200M"]).cuda().eval()
    else:
        pol = vima_b200.VIMAGatoPolicy(**synth.GATO_CFGS[a.model or "gato_200M"]).cuda().eval()
    E, S, Lp = pol.embed_dim, a.slots, a.prompt_len
    Q = a.n_obj if vima else pol._obj_xf_num_queries
    prefix = 0 if vima else Lp + 1
    Lmax = prefix + a.max_steps * (Q + 1)
    pages = lambda cols: -(-cols // 64)  # noqa: E731
    worst = pages(Lmax)  # an episode's pages at its longest
    lengths = np.random.default_rng(a.seed).integers(1, a.max_steps + 1, size=a.episodes).tolist()
    total_steps = int(sum(lengths))
    peak = max(pages_per_tick(lengths, S, Q, prefix))
    pool_tokens = a.kv_pool_tokens or peak // 2 * 64
    # inputs: episode e's k-th step reads bank row (7e + k) % N, its prompt is bank prompt e % P; both runs see the same
    g = torch.Generator(device="cuda").manual_seed(a.seed)
    N, P = 61, 8
    obs_bank = torch.randn(N, Q, E, device="cuda", generator=g)
    msk_bank = torch.rand(N, Q, device="cuda", generator=g) > 0.1
    msk_bank[:, 0] = True
    prompts = torch.randn(Lp, P, E, device="cuda", generator=g)
    pmask = torch.ones(P, Lp, dtype=torch.bool, device="cuda")
    info = gpu_info()
    open_slots = (lambda: pol.open_slots(S, max_tokens=Lmax, max_prompt_tokens=Lp, kv_pool_tokens=pool_tokens)) if vima else \
        (lambda: pol.open_slots(S, max_tokens=Lmax, kv_pool_tokens=pool_tokens))
    print(f"# {info}; policy {a.policy}, model {a.model or ('200M' if vima else 'gato_200M')}, {S} slots, Q={Q}, Lp={Lp}, {a.precision}; "
          f"{a.episodes} episodes of 1..{a.max_steps} steps ({total_steps} env-steps, seed {a.seed}); {Lmax} cache columns per slot; "
          f"history pool {pages(pool_tokens)} pages, the schedule's peak {peak}", flush=True)

    def admit(cache, slots, eps):
        idx = torch.tensor([e % P for e in eps], device="cuda")
        pol.admit(cache, slots, prompts[:, idx].contiguous(), pmask[idx].contiguous())

    def act(cache, rows):
        idx = torch.tensor(rows, device="cuda")
        obs = obs_bank[idx].unsqueeze(0)
        r = pol.act_slots(cache, obs, msk_bank[idx].unsqueeze(0)) if vima else pol.act_slots(cache, obs)
        return torch.cat([r[0][k][0] for k in sorted(r[0])], dim=1)

    def run(mode, record):
        """-> (ticks, stats); record[(episode, k)] = actions of the episode's k-th step (on the device) when record is a dict."""
        cache = open_slots()
        queue = list(range(len(lengths)))
        ep_of = [None] * S       # episode in each slot
        done = {}                # steps taken by each started episode
        parked = []              # (episode, SwappedEpisode, swap call id), oldest episode first
        calls, live_pinned, peak_pinned = {}, 0, 0
        ev_out, ev_in = [], []
        out_bytes = in_bytes = preempt = ticks = 0
        acts = []
        while queue or parked or any(e is not None for e in ep_of):
            free = [b for b in range(S) if ep_of[b] is None]
            if mode == "swap":
                # resume the oldest parked episode while its pages and its next step still fit beside the running ones' next step
                while (parked and free and parked[0][1].prompt_pages <= cache.prompt_pages_free and
                       parked[0][1].kv_pages + pages(Q + 1) <= cache.kv_pages_free - cache.kv_pages_needed(Q)):
                    e, ep, cid = parked.pop(0)
                    b = free.pop(0)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    pol.swap_in(cache, [b], [ep])
                    e1.record()
                    ev_in.append((e0, e1))
                    in_bytes += ep.nbytes
                    ep_of[b] = e
                    calls[cid][1] -= 1
                    if not calls[cid][1]:
                        live_pinned -= calls.pop(cid)[0]
            take = []
            if mode == "reserve":
                budget = cache.kv_pages_total - sum(worst for e in ep_of if e is not None)
                while queue and free and budget >= worst:
                    take.append((free.pop(0), queue.pop(0)))
                    budget -= worst
            elif not parked:
                room = cache.kv_pages_free
                while queue and free and pages(prefix + Q + 1) <= room:  # the prefix and the first step
                    take.append((free.pop(0), queue.pop(0)))
                    room -= pages(prefix + Q + 1)
            if take:
                admit(cache, [b for b, _ in take], [e for _, e in take])
                for b, e in take:
                    ep_of[b], done[e] = e, 0
            if mode == "swap":
                while cache.kv_pages_needed(Q) > cache.kv_pages_free:
                    b = max((b for b in range(S) if ep_of[b] is not None), key=lambda b: ep_of[b])
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    (ep,) = pol.swap_out(cache, [b])
                    e1.record()
                    ev_out.append((e0, e1))
                    cid = len(ev_out)
                    calls[cid] = [ep.nbytes, 1]
                    live_pinned += ep.nbytes
                    peak_pinned = max(peak_pinned, live_pinned)
                    out_bytes += ep.nbytes
                    preempt += 1
                    parked.append((ep_of[b], ep, cid))
                    parked.sort(key=lambda x: x[0])
                    ep_of[b] = None
            active = [b for b in range(S) if ep_of[b] is not None]
            rows = [(7 * ep_of[b] + done[ep_of[b]]) % N if ep_of[b] is not None else 0 for b in range(S)]
            out = act(cache, rows)
            ticks += 1
            if record is not None:
                acts.append((out, [(b, ep_of[b], done[ep_of[b]]) for b in active]))
            ended = []
            for b in active:
                done[ep_of[b]] += 1
                if done[ep_of[b]] == lengths[ep_of[b]]:
                    ended.append(b)
                    ep_of[b] = None
            if ended:
                pol.release(cache, ended)
        torch.cuda.synchronize()
        if record is not None:
            for out, who in acts:
                for b, e, k in who:
                    record[(e, k)] = out[b]
        ms = lambda evs: sum(x.elapsed_time(y) for x, y in evs)  # noqa: E731
        return ticks, {"preemptions": preempt, "swap_out_bytes": out_bytes, "swap_in_bytes": in_bytes,
                       "swap_out_GBps": round(out_bytes / ms(ev_out) / 1e6, 2) if ev_out else None,
                       "swap_in_GBps": round(in_bytes / ms(ev_in) / 1e6, 2) if ev_in else None,
                       "swap_out_ms_total": round(ms(ev_out), 2), "swap_in_ms_total": round(ms(ev_in), 2),
                       "peak_pinned_host_bytes": peak_pinned}

    with torch.no_grad():
        # warm-up: modules, weight packing, kernel attributes, one swap round trip
        c = open_slots()
        n_w = min(S, c.kv_pages_total // pages(prefix + 2 * Q + 2))
        admit(c, list(range(n_w)), list(range(n_w)))
        for _ in range(2):
            act(c, [0] * S)
        pol.swap_in(c, [0], pol.swap_out(c, [0]))
        del c
        torch.cuda.synchronize()
        recs = {}
        for rnd in range(a.rounds):
            for mode in ("reserve", "swap"):
                rec = {} if (a.check and rnd == 0) else None
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                t0 = time.perf_counter()
                ticks, st = run(mode, rec)
                dt = time.perf_counter() - t0
                r = {"run": mode, "round": rnd, "seconds": round(dt, 4), "ticks": ticks, "env_steps_per_s": round(total_steps / dt, 1),
                     "episodes_per_s": round(len(lengths) / dt, 2), **st, "kv_pool_pages": pages(pool_tokens), "schedule_peak_pages": peak,
                     "max_memory_allocated": torch.cuda.max_memory_allocated(), "gpu": info}
                print(json.dumps(r), flush=True)
                if rec is not None:
                    recs[mode] = rec
        if a.check:
            x, y = recs["reserve"], recs["swap"]
            assert len(x) == total_steps and x.keys() == y.keys(), (len(x), len(y))
            bad = [k for k in x if not torch.equal(x[k], y[k])]
            assert not bad, f"{len(bad)} episode steps differ, e.g. {bad[:5]}"
            print(json.dumps({"check": "ok", "episode_steps_compared": len(x)}), flush=True)


if __name__ == "__main__":
    main()
