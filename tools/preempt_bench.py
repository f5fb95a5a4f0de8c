"""Preemption on an overcommitted K/V pool: three drivers of the same episode schedule, alternated in one process.

The schedule is slot_decode_bench.py's: --episodes episodes of 1..--max-steps environment steps (seeded), --slots slots, cfg3 shapes
by default (VIMA-200M, Q = 32 obs tokens, Lp = 256, f16f8); `--policy gato` runs cfg5 (VIMA-Gato-200M, prompt and separator in
the history cache).  Every step is a greedy act_slots.  The history pool holds --kv-pool-tokens tokens, by default half the
schedule's peak page count, so it cannot hold every episode at its longest:

  reserve   admit an episode only when the pool has room for its worst case (--max-steps steps) on top of what the running
            episodes may still take: never refused, never preempted, but fewer episodes run at once
  swap      admit when the episode's prefix and first step fit; before each tick, while the step needs more pages than are free, swap out the
            most recently admitted active episode (policy.swap_out, to pinned host memory); swapped episodes are resumed
            (policy.swap_in), oldest first, before any new episode is admitted
  recompute preempt as `swap` does but with policy.release alone, keeping each parked episode's record on the device (the bank
            rows of its observations and the actions it took); parked episodes are resumed oldest first, before any new episode is
            admitted, by policy.admit_history from that record (action tokens from forward_action_token of the recorded actions),
            as many per call as fit

Each run reports env-steps/s and episodes/s, ticks, preemptions, bytes swapped each way, the swap-out and swap-in rates (bytes over
the CUDA-event time of the swap calls), the peak pinned host bytes held by parked episodes and torch.cuda.max_memory_allocated.
An episode's k-th step takes the same inputs in both runs, so with --check the tool asserts that every episode's per-step actions
in `swap` equal those in `reserve`, and reports the number of episode steps whose actions in `recompute` differ from `reserve`
(recomputed K/V match the stepped ones within the bars of forward_step, not bit for bit, so a near-tied greedy choice can flip).
`recompute` also reports the CUDA-event time of its admit_history calls, the history rows they ran (episodes x padded length) and
the peak device bytes of the parked records.  Weights are random (timing only).  Prints the GPU's name and power limit beside the numbers,
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
    ap.add_argument("--rounds", type=int, default=2, help="each round runs the drivers in turn")
    ap.add_argument("--modes", default="reserve,swap,recompute", help="drivers of each round, in order")
    ap.add_argument("--check", action="store_true", help="assert that swap takes the actions of reserve in every episode; count the "
                                                         "episode steps where recompute does not")
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

    widths = {}  # action key -> head count, in sorted key order (the columns of act's result)

    def act(cache, rows):
        idx = torch.tensor(rows, device="cuda")
        obs = obs_bank[idx].unsqueeze(0)
        r = pol.act_slots(cache, obs, msk_bank[idx].unsqueeze(0)) if vima else pol.act_slots(cache, obs)
        if not widths:
            widths.update({k: r[0][k].shape[-1] for k in sorted(r[0])})
        return torch.cat([r[0][k][0] for k in sorted(r[0])], dim=1)

    def resume(cache, slots, eps, done, recs):
        """admit_history of parked episodes eps (done[e] steps each, recs[e] their action rows) into slots: one call."""
        k = [done[e] for e in eps]
        T = max(max(k), 1)
        rows = torch.tensor([[(7 * e + t) % N if t < kk else 0 for e, kk in zip(eps, k)] for t in range(T)], device="cuda")
        n_act = sum(widths.values())
        zero = torch.zeros(n_act, dtype=torch.int64, device="cuda")
        acts = torch.stack([torch.stack(recs.get(e, []) + [zero] * (T - len(recs.get(e, [])))) for e in eps], 1)  # (T, n, n_act)
        d, c0 = {}, 0
        for key, w in widths.items():
            d[key] = acts[..., c0:c0 + w]
            c0 += w
        at = pol.forward_action_token(d)
        idx = torch.tensor([e % P for e in eps], device="cuda")
        pt, pm = prompts[:, idx].contiguous(), pmask[idx].contiguous()
        if vima:
            pol.admit_history(cache, slots, pt, pm, obs_bank[rows], msk_bank[rows], at, k)
        else:
            pol.admit_history(cache, slots, pt, pm, obs_bank[rows], at, k)

    def run(mode, record):
        """-> (ticks, stats); record[(episode, k)] = actions of the episode's k-th step (on the device) when record is a dict."""
        cache = open_slots()
        queue = list(range(len(lengths)))
        ep_of = [None] * S       # episode in each slot
        done = {}                # steps taken by each started episode
        parked = []              # (episode, SwappedEpisode, swap call id), oldest episode first; recompute: (episode, None, None)
        calls, live_pinned, peak_pinned = {}, 0, 0
        ev_out, ev_in, ev_re = [], [], []
        out_bytes = in_bytes = preempt = ticks = 0
        recs, rec_bytes, peak_rec, re_rows, re_eps = {}, 0, 0, 0, 0  # recompute: each started episode's action rows on the device
        n_act = sum(widths.values()) * 8
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
            if mode == "recompute":
                group = []
                room = cache.kv_pages_free - cache.kv_pages_needed(Q)
                proom = cache.prompt_pages_free
                while parked and free:
                    e = parked[0][0]
                    need = pages(prefix + (done[e] * (Q + 1) - 1 if done[e] else 0) + Q + 1)  # its history and its next step
                    if need > room or (vima and pages(Lp) > proom):
                        break
                    parked.pop(0)
                    group.append((free.pop(0), e))
                    room -= need
                    proom -= pages(Lp) if vima else 0
                if group:
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    resume(cache, [b for b, _ in group], [e for _, e in group], done, recs)
                    e1.record()
                    ev_re.append((e0, e1))
                    re_rows += len(group) * max(prefix + (done[e] * (Q + 1) - 1 if done[e] else 0) for _, e in group)
                    re_eps += len(group)
                    for b, e in group:
                        ep_of[b] = e
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
            if mode == "recompute":
                while cache.kv_pages_needed(Q) > cache.kv_pages_free:
                    b = max((b for b in range(S) if ep_of[b] is not None), key=lambda b: ep_of[b])
                    pol.release(cache, [b])
                    preempt += 1
                    parked.append((ep_of[b], None, None))
                    parked.sort(key=lambda x: x[0])
                    ep_of[b] = None
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
                if mode == "recompute":
                    recs.setdefault(ep_of[b], []).append(out[b])
                    rec_bytes += n_act
                done[ep_of[b]] += 1
                if done[ep_of[b]] == lengths[ep_of[b]]:
                    ended.append(b)
                    if mode == "recompute":
                        rec_bytes -= n_act * len(recs.pop(ep_of[b]))
                    ep_of[b] = None
            peak_rec = max(peak_rec, rec_bytes)
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
                       "peak_pinned_host_bytes": peak_pinned, "admit_history_ms_total": round(ms(ev_re), 2),
                       "resumed_episodes": re_eps, "recomputed_rows": re_rows, "peak_record_device_bytes": peak_rec}

    with torch.no_grad():
        # warm-up: modules, weight packing, kernel attributes, one swap round trip
        c = open_slots()
        n_w = min(S, c.kv_pages_total // pages(prefix + 2 * Q + 2))
        admit(c, list(range(n_w)), list(range(n_w)))
        for _ in range(2):
            act(c, [0] * S)
        pol.swap_in(c, [0], pol.swap_out(c, [0]))
        pol.release(c, [0])
        resume(c, [0], [0], {0: 2}, {0: [act(c, [0] * S)[0]] * 2})
        del c
        torch.cuda.synchronize()
        recs = {}
        for rnd in range(a.rounds):
            for mode in a.modes.split(","):
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
            x = recs["reserve"]
            assert len(x) == total_steps, len(x)
            if "swap" in recs:
                y = recs["swap"]
                assert x.keys() == y.keys(), (len(x), len(y))
                bad = [k for k in x if not torch.equal(x[k], y[k])]
                assert not bad, f"{len(bad)} episode steps differ, e.g. {bad[:5]}"
                print(json.dumps({"check": "ok", "run": "swap", "episode_steps_compared": len(x)}), flush=True)
            if "recompute" in recs:
                y = recs["recompute"]
                assert x.keys() == y.keys(), (len(x), len(y))
                bad = [k for k in x if not torch.equal(x[k], y[k])]
                print(json.dumps({"check": "counted", "run": "recompute", "episode_steps_compared": len(x), "episode_steps_differing": len(bad),
                                  "episodes_differing": len({e for e, _ in bad})}), flush=True)


if __name__ == "__main__":
    main()
