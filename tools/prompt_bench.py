"""Prompt encode (VIMAPolicy.forward_prompt_assembly: word / object embeddings, 12-layer T5, post layer) at B = 256 for cfg3's prompt
(Lp = 256), a 384-token and a real 512-token prompt (480 words + one image of 32 object tokens, the shape of bench.py's cfg3x).

    python tools/prompt_bench.py [--batch 256] [--precision f16f8] [--reps 20] [--warmup 3] [--no-reference]

Reports, one JSON line each:
  * e2e       ms per batch and prompts/s, CUDA events around each of --reps calls after --warmup (median);
  * kernels   a separate torch.profiler run: device time of the attention kernels per batch and their share of all kernel time;
  * at Lp = 256 and 384 both with attn_bias=auto (the resident-K/V mma.sync kernel) and attn_bias=tc (the K/V-streaming wgmma kernel);
  * reference when oracle/_ref is staged: the unmodified reference's forward_prompt_assembly in eager PyTorch fp32 on the same GPU at
    Lp = 512 (same weights and inputs), its time, and the rel-L2 of our prompt tokens against it.
The GPU's name and power limit are printed with the numbers.  Weights come from oracle.detgen (needed for the reference comparison).
"""
import argparse
import dataclasses
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import vima_b200  # noqa: E402
from oracle import detgen, synth  # noqa: E402


def gpu_info() -> str:
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[torch.cuda.current_device()]
    except Exception:  # noqa: BLE001 -- the name alone is still worth printing
        return f"{torch.cuda.get_device_name()}, power limit not readable"


def cases(batch):
    base = dataclasses.replace(synth.CASES["cfg3"], B=batch)
    return {256: base, 384: dataclasses.replace(base, name="prompt384", n_words=352, seed=19),
            512: dataclasses.replace(base, name="cfg3x", n_words=480, seed=18)}


def to_dev(x, dev):
    return {k: to_dev(v, dev) for k, v in x.items()} if isinstance(x, dict) else x.to(dev)


def prompt_inputs(case, dev, DataDict):
    token_types, words, images = synth.make_prompt(case)
    return token_types, words.to(dev), DataDict(to_dev(images, dev))


def time_calls(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return statistics.median(ms), (max(ms) - min(ms)) / statistics.median(ms)


def kernel_times(fn, reps):
    """-> (attention kernel ms per call, all kernel ms per call, {attention kernel name: ms per call})."""
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    total, attn = 0.0, {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        us = ev.time_range.elapsed_us()
        total += us
        if "attention" in ev.name:
            name = ev.name.replace("(anonymous namespace)::", "").split("(")[0].split("<")[0].replace("void ", "").replace("vima::", "")
            attn[name] = attn.get(name, 0.0) + us
    return sum(attn.values()) / 1e3 / reps, total / 1e3 / reps, {k: v / 1e3 / reps for k, v in attn.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--precision", default="f16f8")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-reference", action="store_true")
    args = ap.parse_args()

    from vima_b200 import _C
    from vima_b200.utils import DataDict

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    card = gpu_info()
    vima_b200.set_precision(args.precision)
    ctx = _C.Context.get(dev)
    cfg = synth.MODEL_CFGS["200M"]
    pol = vima_b200.VIMAPolicy(**cfg)
    detgen.fill_module_(pol)
    pol = pol.to(dev).eval()
    runs = [(256, "auto"), (256, "tc"), (384, "auto"), (384, "tc"), (512, "auto")]
    ours512 = None
    with torch.no_grad():
        for Lp, attn_bias in runs:
            case = cases(args.batch)[Lp]
            inp = prompt_inputs(case, dev, DataDict)
            ctx.set_option("attn_bias", attn_bias)
            fn = lambda: pol.forward_prompt_assembly(inp)  # noqa: E731
            ms, spread = time_calls(fn, args.reps, args.warmup)
            attn_ms, kern_ms, per_kernel = kernel_times(fn, max(3, args.reps // 4))
            tok, msk = fn()
            assert tok.shape[0] == Lp, tok.shape
            if Lp == 512:
                ours512 = tok.float().cpu()
            print(json.dumps({"what": "prompt_encode", "Lp": Lp, "B": args.batch, "precision": args.precision, "attn_bias": attn_bias,
                              "ms_per_batch": round(ms, 3), "spread": round(spread, 3), "prompts_per_s": round(args.batch / ms * 1e3, 1),
                              "reps": args.reps, "attention_ms": round(attn_ms, 3), "kernel_ms": round(kern_ms, 3),
                              "attention_share": round(attn_ms / kern_ms, 4), "attention_kernels_ms": {k: round(v, 3) for k, v in per_kernel.items()},
                              "gpu": card}), flush=True)
    ctx.set_option("attn_bias", "auto")
    del pol
    torch.cuda.empty_cache()

    from oracle.ref_shim import reference_available

    if args.no_reference or not reference_available():
        print(json.dumps({"what": "reference", "status": "not measured (oracle/_ref not staged)" if not args.no_reference else "skipped"}))
        return
    from oracle.ref_shim import load_reference

    ref = load_reference()
    RDD = sys.modules["vima.utils"].DataDict
    torch.manual_seed(0)
    rpol = ref.VIMAPolicy(**cfg)
    detgen.fill_module_(rpol)
    rpol = rpol.to(dev).eval()
    case = cases(args.batch)[512]
    inp = prompt_inputs(case, dev, RDD)
    with torch.no_grad():
        fn = lambda: rpol.forward_prompt_assembly(inp)  # noqa: E731
        ms, spread = time_calls(fn, max(3, args.reps // 4), 1)
        rtok, _ = fn()
    rtok = rtok.float().cpu()
    err = ((ours512.double() - rtok.double()).norm() / rtok.double().norm()).item()
    print(json.dumps({"what": "reference_prompt_encode", "Lp": 512, "B": args.batch, "impl": "unmodified reference, eager PyTorch fp32",
                      "ms_per_batch": round(ms, 3), "spread": round(spread, 3), "prompts_per_s": round(args.batch / ms * 1e3, 1),
                      "rel_l2_ours_vs_reference": err, "our_precision": args.precision, "gpu": card}), flush=True)


if __name__ == "__main__":
    main()
