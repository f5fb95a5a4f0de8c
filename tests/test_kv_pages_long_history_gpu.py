"""GPU: the staggered slot runs of test_long_history_gpu.py (VIMA-Gato and VIMAPolicy at n_positions = 1024, past 768 tokens) on a
K/V page pool smaller than S * Lmax that their schedules fit, free list shuffled: every active slot's row equals the default
pool's bit for bit at every tick."""
import random

import pytest
import torch

from tests.test_long_history_gpu import GATO_ADMITS, GATO_RELEASES, GATO_TICKS, _pad_cat, _rand_prompt, gato_policy, vima_policy

pytestmark = pytest.mark.gpu


def _run(pol, cache, S, ticks, admits, releases, seed, vima, peak):
    g = torch.Generator(device="cuda").manual_seed(seed)
    E = pol.embed_dim
    Q = 32 if vima else pol._obj_xf_num_queries
    outs = []
    for t in range(ticks):
        for b in releases.get(t, []):
            pol.release(cache, [b])
        if t in admits:
            slots = sorted(admits[t])
            pol.admit(cache, slots, *_pad_cat([_rand_prompt(g, admits[t][b], E) for b in slots]))
        obs = torch.randn(1, S, Q, E, device="cuda", generator=g)
        act = torch.randn(1, S, E, device="cuda", generator=g)
        if vima:
            msk = torch.rand(1, S, Q, device="cuda", generator=g) > 0.2
            msk[..., 0] = True
            out = pol.step_slots(cache, obs, msk, act)
        else:
            out = pol.step_slots(cache, obs, act)
        peak.append(cache.kv_pages_total - cache.kv_pages_free)
        outs.append(out[:, [b for b in range(S) if cache.active_host[b]]].clone())
    torch.cuda.synchronize()
    return outs


@pytest.mark.parametrize("mode", ["f16x3", "f16f8"])
@pytest.mark.parametrize("kind", ["gato", "vima"])
def test_long_history_slots_on_a_small_pool(kind, mode):
    import vima_b200

    vima_b200.set_precision(mode)
    try:
        vima = kind == "vima"
        pol = vima_policy() if vima else gato_policy()
        if vima:
            S, ticks, admits, releases = 3, 28, {0: {0: 40, 2: 17}, 3: {1: 25}}, {20: [2]}
            open_ = lambda pool=None: pol.open_slots(S, max_prompt_tokens=64, kv_pool_tokens=pool)  # noqa: E731
        else:
            S, ticks, admits, releases = 4, GATO_TICKS, GATO_ADMITS, GATO_RELEASES
            open_ = lambda pool=None: pol.open_slots(S, kv_pool_tokens=pool)  # noqa: E731
        with torch.no_grad():
            peak = []
            c0 = open_()
            ref = _run(pol, c0, S, ticks, admits, releases, 7, vima, peak)
            assert max(c0.len_host) > 768 and max(peak) < c0.kv_pages_total
            c1 = open_(64 * max(peak))
            random.Random(3).shuffle(c1.pages.free)
            got = _run(pol, c1, S, ticks, admits, releases, 7, vima, [])
        for t, (a, b) in enumerate(zip(ref, got)):
            assert torch.equal(a, b), (kind, mode, t)
    finally:
        vima_b200.set_precision("f16x3")
