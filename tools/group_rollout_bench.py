"""Group sampling: k rollouts of one episode, as k independent admissions against one admission plus fork_slots.

256 slots in 32 blocks of k = 8.  Each block runs one group at a time: k rollouts of the same episode (same prompt, same
observations here) that act with an ActionSampler, so they draw different actions, and end at their own lengths (1..15 environment
steps, seeded).  A member that ends is released; when the whole group has ended the block takes the next group.  Two arms, each
eager (act_slots) and replayed from one CUDA graph (capture_act_slots), alternated (a, b, a, b) in one process:

  (a) admit    the group's prompt admitted into all k slots of the block
  (b) fork     the prompt admitted into the block's first slot, then fork_slots(cache, [first] * (k - 1), the other k - 1)

Sizes: cfg3 (VIMA-200M, Q = 32 obs tokens, Lp = 256, f16f8) and cfg5 shapes (VIMA-Gato-200M, Q = 16, Lp = 256: 257 prefill rows in
the self-attention cache).  Reported per run: env-steps/s, admission time per episode (CUDA events around the admit / fork calls,
on the stream the steps run on), peak K/V pages in use, and the smallest pool the arm's schedule fits (the host allocator's peak,
read after each step's reservation); for cfg3 also the peak prompt pages and the smallest prompt pool (the fork arm's forks share
their source's prompt pages), and torch.cuda.max_memory_allocated over the run.  --prompt-pool-tokens opens cfg3's caches with that
prompt pool (default: room for a full-length prompt in every slot).  Weights are random (timing only).  Prints the GPU's name and
power limit beside the numbers, one JSON line per run.
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
from rollout_bench import gpu_info  # card name and power limit


def make_policy(size):
    if size == "cfg3":
        pol = vima_b200.VIMAPolicy(**synth.MODEL_CFGS["200M"])
    else:
        pol = vima_b200.VIMAGatoPolicy(**synth.GATO_CFGS["gato_200M"])
    return pol.cuda().eval()


def run_size(size, a, info):
    pol = make_policy(size)
    vima = size == "cfg3"
    S, k, Lp = a.slots, a.group, a.prompt_len
    E = pol.embed_dim
    Q = a.n_obj if vima else pol._obj_xf_num_queries
    pre = 0 if vima else Lp + 1
    Lmax = pre + a.max_steps * (Q + 1)
    n_blocks = S // k
    rng = np.random.default_rng(a.seed)
    lengths = rng.integers(1, a.max_steps + 1, size=(a.groups, k)).tolist()
    total_steps = int(sum(map(sum, lengths)))
    g = torch.Generator(device="cuda").manual_seed(a.seed)
    obs_pool = [torch.randn(1, S, Q, E, device="cuda", generator=g) for _ in range(3)]
    msk = torch.rand(1, S, Q, device="cuda", generator=g) > 0.1
    msk[..., 0] = True
    prompts = torch.randn(Lp, n_blocks, E, device="cuda", generator=g)
    pmask = torch.ones(n_blocks, Lp, dtype=torch.bool, device="cuda")
    extra = (msk,) if vima else ()
    if vima:
        open_slots = lambda: pol.open_slots(S, max_tokens=Lmax, max_prompt_tokens=Lp, prompt_pool_tokens=a.prompt_pool_tokens)  # noqa: E731
    else:
        open_slots = lambda: pol.open_slots(S, max_tokens=Lmax)  # noqa: E731
    print(f"# {info}; {size} ({type(pol).__name__}), {S} slots in groups of {k}, Q={Q}, Lp={Lp}, {a.precision}; {a.groups} groups "
          f"({a.groups * k} episodes of 1..{a.max_steps} steps, {total_steps} env-steps, seed {a.seed})", flush=True)

    def start_groups(cache, arm, blocks):
        """Admit the next group into each block of `blocks` (prompt of block j = column j)."""
        if arm == "admit":
            slots = [j * k + i for j in blocks for i in range(k)]
            pol.admit(cache, slots, prompts[:, blocks].repeat_interleave(k, dim=1), pmask[blocks].repeat_interleave(k, dim=0))
        else:
            pol.admit(cache, [j * k for j in blocks], prompts[:, blocks], pmask[blocks])
            pol.fork_slots(cache, [j * k for j in blocks for _ in range(k - 1)], [j * k + i for j in blocks for i in range(1, k)])

    def run(cache, arm, step):
        queue = list(range(a.groups))
        remaining = [0] * S
        ticks, idle_blocks, peak, peak_p, admits = 0, list(range(n_blocks)), 0, 0, []
        while True:
            take = idle_blocks[:len(queue)]
            if take:
                ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
                ev[0].record()
                start_groups(cache, arm, take)
                ev[1].record()
                admits.append((ev, len(take) * k))
                peak_p = max(peak_p, cache.prompt_pages_total - cache.prompt_pages_free)
                for j in take:
                    for i, n in enumerate(lengths[queue.pop(0)]):
                        remaining[j * k + i] = n
            if not any(remaining):
                break
            step(cache, obs_pool[ticks % 3])
            peak = max(peak, cache.kv_pages_total - cache.kv_pages_free)
            ticks += 1
            ended = []
            for b in range(S):
                if remaining[b]:
                    remaining[b] -= 1
                    if remaining[b] == 0:
                        ended.append(b)
            if ended:
                pol.release(cache, ended)
            idle_blocks = [j for j in range(n_blocks) if not any(remaining[j * k:(j + 1) * k])]
        torch.cuda.synchronize()
        adm_ms = sum(e[0].elapsed_time(e[1]) for e, _ in admits)
        return ticks, peak, peak_p, adm_ms, sum(n for _, n in admits)

    with torch.no_grad():
        c = open_slots()  # warm-up: modules, weight packing, kernel attributes
        warm = vima_b200.ActionSampler(a.seed, "cuda")
        for arm in ("admit", "fork"):
            start_groups(c, arm, list(range(n_blocks)))
            for _ in range(2):
                pol.act_slots(c, obs_pool[0], *extra, sampler=warm)
        del c
        torch.cuda.synchronize()
        for rnd in range(a.rounds):
            for mode in ("eager", "graph"):
                for arm in ("admit", "fork"):
                    cache = open_slots()
                    sampler = vima_b200.ActionSampler(a.seed, "cuda")
                    info_run = {}
                    if mode == "eager":
                        step = lambda c, o: pol.act_slots(c, o, *extra, sampler=sampler)  # noqa: E731
                    else:
                        start_groups(cache, arm, list(range(n_blocks)))
                        t0 = time.perf_counter()
                        gs = pol.capture_act_slots(cache, obs_pool[0], *extra, sampler=sampler)
                        torch.cuda.synchronize()
                        info_run = {"capture_s": round(time.perf_counter() - t0, 3)}
                        pol.release(cache, list(range(S)))
                        step = lambda c, o: gs(o, *extra)  # noqa: E731
                    torch.cuda.synchronize()
                    torch.cuda.reset_peak_memory_stats()
                    t0 = time.perf_counter()
                    ticks, peak, peak_p, adm_ms, n_adm = run(cache, arm, step)
                    dt = time.perf_counter() - t0
                    r = {"size": size, "slots": S, "group": k, "arm": arm, "mode": mode, "round": rnd, "seconds": round(dt, 4),
                         "ticks": ticks, "env_steps_per_s": round(total_steps / dt, 1), "ms_per_tick": round(dt * 1e3 / ticks, 3),
                         "admission_ms_per_episode": round(adm_ms / n_adm, 4), "peak_pages": peak, "min_pool_tokens": peak * 64,
                         "pool_pages_default": cache.kv_pages_total, "max_memory_allocated_gb": round(torch.cuda.max_memory_allocated() / 1e9, 3)}
                    if vima:
                        r.update({"peak_prompt_pages": peak_p, "min_prompt_pool_tokens": peak_p * 64, "prompt_pool_pages": cache.prompt_pages_total})
                    r.update(info_run)
                    r["gpu"] = info
                    print(json.dumps(r), flush=True)
                    del cache
    del pol
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="cfg3,cfg5")
    ap.add_argument("--slots", type=int, default=256)
    ap.add_argument("--group", type=int, default=8)
    ap.add_argument("--groups", type=int, default=96)
    ap.add_argument("--n-obj", type=int, default=32)
    ap.add_argument("--prompt-len", type=int, default=256)
    ap.add_argument("--max-steps", type=int, default=15)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--precision", default="f16f8")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--prompt-pool-tokens", type=int, default=None, help="cfg3: prompt pool size (default: every slot a full prompt)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("group_rollout_bench needs a CUDA device")
    vima_b200.set_precision(a.precision)
    torch.manual_seed(a.seed)
    info = gpu_info()
    for size in a.sizes.split(","):
        run_size(size, a, info)


if __name__ == "__main__":
    main()
