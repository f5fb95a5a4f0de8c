"""GPU: packed weights, captured graphs and decode caches follow a weight update -- or refuse to run on the old weights.

Every fast path keeps state derived from the parameters: the packed-weight caches (engine.WeightCache), the device pointers baked
into a captured graph (graphs.GraphedStep / GraphedSlotStep) and the K/V rows of an open decode cache.  Here the weights of a
live policy change after its first step by every supported route, and:
  * the next eager step equals a cold recompute (the same policy after every packed-weight cache in its tree was cleared) bit for
    bit, and differs from the step before; one case per policy kind also meets the CPU oracle run with the new state dict;
  * perturbing any single parameter changes the step, and the warm step still equals the cold one (no cache key misses a parameter,
    no parameter is ignored by the CUDA path);
  * a captured graph refuses to replay (RuntimeError, nothing launched) and a fresh capture equals the eager step;
  * an open decode cache refuses to step or admit (ValueError, state unchanged), and a new one matches the full re-forward.
The kernels are deterministic, so "equal" is torch.equal throughout."""
import time

import pytest
import torch
import torch.nn as nn

from oracle import detgen, synth, vima_oracle as O
from tests.policy_runner import to_dev
from tests.util import rel_l2

pytestmark = pytest.mark.gpu

VIMA_CASES = {"vima2M": synth.CASES["cfg1_t2"], "vima4M": synth.CASES["ragged_4M"]}
KINDS = ["vima2M", "vima4M", "gato", "gpt", "flamingo"]
ROUTES = ["load_state_dict", "load_state_dict_assign", "inplace_no_grad", "data_assign", "new_parameter", "data_copy_refresh"]
SEED2 = 1  # the second deterministic weight set (detgen seed)

_POL = {}


@pytest.fixture(autouse=True)
def _precision_reset():
    yield
    import vima_b200

    vima_b200.set_precision("f16x3")


def _clear_caches(pol):
    """Cold start: every packed-weight cache in the module tree emptied (what refresh_weights does, spelled out here)."""
    for m in pol.modules():
        if "_wc" in m.__dict__:
            m._wc.clear()


def _sd(pol, seed):
    sd = {}
    for k, v in pol.state_dict().items():
        w = detgen.weight_for(k, v.shape, seed)
        sd[k] = v.detach().cpu().clone() if w is None else w.to(v.dtype)
    return sd


def _policy(kind):
    """The policy of `kind` with the seed-0 weights, plus the seed-0 / seed-1 state dicts (CPU).  One policy object per kind for
    the whole module; every call puts the seed-0 weights back into new parameters, so no test sees another's updates."""
    import vima_b200

    if kind not in _POL:
        if kind.startswith("vima"):
            pol = vima_b200.VIMAPolicy(**synth.MODEL_CFGS[VIMA_CASES[kind].model])
        else:
            cls = {"gato": vima_b200.VIMAGatoPolicy, "gpt": vima_b200.VIMAGPTPolicy, "flamingo": vima_b200.VIMAFlamingoPolicy}[kind]
            pol = cls(**(synth.FLAMINGO_CFGS["flamingo_tiny"] if kind == "flamingo" else synth.GATO_CFGS["gato_tiny"]))
        pol = pol.cuda().eval()
        _POL[kind] = (pol, _sd(pol, 0), _sd(pol, SEED2))
    pol, sd0, sd1 = _POL[kind]
    pol.load_state_dict({k: v.cuda() for k, v in sd0.items()}, assign=True)
    return pol, sd0, sd1


# ------------------------------------------------------------------------------------------------------------------------------
# the full step: prompt assembly, obs tokens, forward, action decoder, next action token
def _tokens(kind, pol):
    from vima_b200.utils import DataDict

    if kind.startswith("vima"):
        case = VIMA_CASES[kind]
        tt, wb, ib = synth.make_prompt(case)
        pt, pm = pol.forward_prompt_assembly((tt, wb.cuda(), DataDict(to_dev(ib, "cuda"))))
        ot, om = pol.forward_obs_token(DataDict(to_dev(synth.make_obs(case), "cuda")))
        at = pol.forward_action_token(to_dev(synth.make_actions(case, case.T), "cuda"))
        return pt, pm, ot, om, at
    from tests.test_baseline_decode_gpu import _case_tokens

    pt, pm, ot, at = _case_tokens(kind, pol)
    return pt, pm, ot, None, at


def _forward(kind, pol, pt, pm, ot, om, at):
    T = ot.shape[0]
    a = at[:T - 1] if T > 1 else None
    if kind.startswith("vima"):
        return pol.forward(obs_token=ot, obs_mask=om, action_token=a, prompt_token=pt, prompt_token_mask=pm)
    return pol.forward(ot, a, pt, pm)


def _heads(pol, pred):
    dists = pol.forward_action_decoder(pred[-1:])
    raw = torch.cat([dists[k].raw_logits for k in dists], dim=-1)
    modes = {k: v.mode() for k, v in dists.items()}
    return [raw, torch.cat(list(modes.values()), dim=-1), pol.forward_action_token(modes)]


@torch.no_grad()
def _step(kind, pol):
    """Every output of one full step, cloned, in a fixed order."""
    pt, pm, ot, om, at = _tokens(kind, pol)
    pred = _forward(kind, pol, pt, pm, ot, om, at)
    outs = [pt, pm, ot, at, pred] + ([om] if om is not None else []) + _heads(pol, pred)
    torch.cuda.synchronize()
    return [t.clone() for t in outs]


def _cold(kind, pol):
    _clear_caches(pol)
    return _step(kind, pol)


def _equal(a, b):
    return len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b))


def _first_diff(a, b):
    return [i for i, (x, y) in enumerate(zip(a, b)) if not torch.equal(x, y)]


# ------------------------------------------------------------------------------------------------------------------------------
def _parameters(pol):
    """(name, module, attribute) of every parameter, aliases included (a tied tensor is updated under each of its names)."""
    out = []
    for mname, m in pol.named_modules(remove_duplicate=False):
        for n, p in m._parameters.items():
            if p is not None:
                out.append((f"{mname}.{n}" if mname else n, m, n))
    return out


@torch.no_grad()
def _update(pol, route, sd):
    """Switch the policy's weights to `sd` (CPU state dict) by `route`."""
    dev = {k: v.cuda() for k, v in sd.items()}
    if route == "load_state_dict":
        pol.load_state_dict(dev)
    elif route == "load_state_dict_assign":
        pol.load_state_dict(dev, assign=True)
    elif route == "inplace_no_grad":  # halve then double: exact for these weights, and two in-place ops on every parameter
        for name, m, n in _parameters(pol):
            getattr(m, n).copy_(dev[name] * 0.5)
        for p in pol.parameters():
            p.mul_(2.0)
    elif route == "data_assign":
        for name, m, n in _parameters(pol):
            getattr(m, n).data = dev[name].clone()
    elif route == "new_parameter":
        for name, m, n in _parameters(pol):
            setattr(m, n, nn.Parameter(dev[name].clone(), requires_grad=False))
    elif route == "data_copy_refresh":
        for p_name, p in pol.named_parameters():
            p.data.copy_(dev[p_name])
        pol.refresh_weights()
    else:
        raise AssertionError(route)


def _check_sd(pol, sd):
    for k, v in pol.state_dict().items():
        assert torch.equal(v.cpu(), sd[k]), k


# ------------------------------------------------------------------------------------------------------------------------------
# 1a. update routes, eager path
@pytest.mark.parametrize("route", ROUTES)
@pytest.mark.parametrize("mode", ["f16x3", "f16f8"])
@pytest.mark.parametrize("kind", KINDS)
def test_update_route_eager_equals_cold(kind, mode, route):
    import vima_b200

    vima_b200.set_precision(mode)
    pol, sd0, sd1 = _policy(kind)
    before = _step(kind, pol)
    assert _equal(_step(kind, pol), before)  # warm caches: same result
    _update(pol, route, sd1)
    _check_sd(pol, sd1)
    after = _step(kind, pol)
    assert not torch.equal(after[4], before[4]), "the step did not change with the weights"
    cold = _cold(kind, pol)
    assert _equal(after, cold), (route, _first_diff(after, cold))


def test_update_route_bf16x3():
    import vima_b200

    vima_b200.set_precision("bf16x3")
    pol, sd0, sd1 = _policy("vima2M")
    before = _step("vima2M", pol)
    _update(pol, "load_state_dict", sd1)
    after = _step("vima2M", pol)
    assert not torch.equal(after[4], before[4])
    cold = _cold("vima2M", pol)
    assert _equal(after, cold), _first_diff(after, cold)


@torch.no_grad()
def _oracle_pred(kind, sd, pt, pm, ot, om, at):
    """The CPU oracle's predicted action tokens and raw logits with state dict `sd` (VIMA: the whole step from the synthetic case;
    baselines: the decoder and heads on the CUDA path's tokens)."""
    if kind.startswith("vima"):
        case = VIMA_CASES[kind]
        cfg = synth.MODEL_CFGS[case.model]
        pt_o, pm_o, _ = O.forward_prompt_assembly(sd, synth.make_prompt(case))
        ot_o, om_o = O.forward_obs_token(sd, synth.make_obs(case))
        at_o = O.forward_action_token(sd, synth.make_actions(case, case.T))
        T = ot_o.shape[0]
        pred = O.policy_forward(sd, ot_o, om_o, at_o[:T - 1] if T > 1 else None, pt_o, pm_o, n_head=cfg["sattn_n_heads"],
                                xattn_n_head=cfg["xattn_n_heads"])
    else:
        from tests.test_baseline_decode_gpu import _oracle

        T = ot.shape[0]
        pred = _oracle(kind, sd, ot, at[:T - 1] if T > 1 else None, pt, pm)
    return pred, O.action_decoder_logits(sd, pred[-1:])


@pytest.mark.parametrize("kind", KINDS)
def test_updated_weights_match_oracle(kind):
    """The cold recompute is itself right: after the update the step meets the CPU oracle run with the new weights."""
    import vima_b200

    vima_b200.set_precision("f16x3")
    pol, sd0, sd1 = _policy(kind)
    _step(kind, pol)
    _update(pol, "load_state_dict", sd1)
    with torch.no_grad():
        pt, pm, ot, om, at = _tokens(kind, pol)
        pred = _forward(kind, pol, pt, pm, ot, om, at)
        raw = _heads(pol, pred)[0]
    want_pred, want_raw = _oracle_pred(kind, sd1, pt, pm, ot, om, at)
    assert rel_l2(want_pred.numpy(), pred.cpu().numpy()) < 1e-3
    assert rel_l2(want_raw.numpy(), raw[-1:].cpu().numpy().reshape(want_raw.shape)) < 1e-3
    old_pred, _ = _oracle_pred(kind, sd0, pt, pm, ot, om, at)
    assert rel_l2(old_pred.numpy(), pred.cpu().numpy()) > 1e-2  # and the old weights would not


# ------------------------------------------------------------------------------------------------------------------------------
# 1b. per-parameter sweep
# parameters the reference's forward never reads, so no step output can move with them
UNUSED = {
    # the T5 token table (also `encoder.embed_tokens`): the prompt encoder takes inputs_embeds (reference
    # vima/nn/prompt_encoder/prompt_encoder.py:52), so the table is never indexed
    "vima2M": {"t5_prompt_encoder.t5.shared.weight"},
    # the same T5 table, and the GPT token table: the decoder takes inputs_embeds (reference vima/nn/seq_modeling/gpt/gpt.py:70)
    "gato": {"t5_prompt_encoder.t5.shared.weight", "transformer.lm.tokens_embed.weight"},
}


@pytest.mark.parametrize("kind", ["vima2M", "gato"])
def test_every_parameter_reaches_the_step(kind):
    import vima_b200

    vima_b200.set_precision("f16x3")
    pol, sd0, sd1 = _policy(kind)
    g = torch.Generator(device="cuda").manual_seed(2024)
    prev = _cold(kind, pol)
    t0 = time.perf_counter()
    unchanged, n = [], 0
    for name, p in list(pol.named_parameters()):
        with torch.no_grad():
            p.add_(0.01 * torch.randn(p.shape, device=p.device, generator=g))
        warm = _step(kind, pol)
        cold = _cold(kind, pol)
        assert _equal(warm, cold), (name, _first_diff(warm, cold))
        if _equal(warm, prev):
            unchanged.append(name)
        prev, n = cold, n + 1
    dt = time.perf_counter() - t0
    print(f"{kind}: {n} parameters swept in {dt:.1f} s")
    assert sorted(unchanged) == sorted(UNUSED[kind]), unchanged


# ------------------------------------------------------------------------------------------------------------------------------
# 1c. graphs
def _graph_step(kind, pol):
    """A GraphedStep-capturable step over new obs inputs (the prompt tokens and history are computed once, as bench.py does)."""
    from vima_b200.utils import DataDict

    with torch.no_grad():
        pt, pm, ot, om, at = _tokens(kind, pol)
    if kind.startswith("vima"):
        case = VIMA_CASES[kind]
        obs = to_dev(synth.slice_obs(synth.make_obs(case), case.T - 1, case.T), "cuda")
    else:
        case = synth.GATO_CASES["gato_small"]
        obs = to_dev(synth.make_gato_obs(case, T=1), "cuda")
    T = ot.shape[0]

    @torch.no_grad()
    def step(obs_dev):
        if kind.startswith("vima"):
            n_tok, n_msk = pol.forward_obs_token(DataDict(obs_dev))
            o = torch.cat([ot[:T - 1], n_tok], 0)
            m = torch.cat([om[:T - 1], n_msk], 0)
        else:
            n_tok = pol.forward_obs_token(DataDict(obs_dev))
            o, m = torch.cat([ot[:T - 1], n_tok], 0), None
        pred = _forward(kind, pol, pt, pm, o, m, at)
        return [pred[-1:]] + _heads(pol, pred)

    return step, obs


def _sentinel(outs):
    for t in outs:
        t.fill_(-12345)
    return lambda: all(bool((t == -12345).all()) for t in outs)


@pytest.mark.parametrize("kind", ["vima2M", "gato"])
def test_graph_refuses_updated_weights(kind):
    import vima_b200
    from vima_b200.graphs import GraphedStep

    vima_b200.set_precision("f16x3")
    pol, sd0, sd1 = _policy(kind)
    step, obs = _graph_step(kind, pol)
    eager = [t.clone() for t in step(obs)]
    g = GraphedStep(step, obs, warmup=2)
    assert _equal(g(obs), eager)
    for route in ("load_state_dict", "load_state_dict_assign", "new_parameter"):
        _update(pol, route, sd1)
        n0 = g.ctx.launches
        still = _sentinel(g.static_out)
        with pytest.raises(RuntimeError, match="[Cc]apture it again"):
            g(obs)
        torch.cuda.synchronize()
        assert g.ctx.launches == n0 and still(), route
        # the original values back, in place: the versions moved, so replay is still refused
        with torch.no_grad():
            for name, m, n in _parameters(pol):
                getattr(m, n).copy_(sd0[name].cuda())
        with pytest.raises(RuntimeError, match="[Cc]apture it again"):
            g(obs)
        torch.cuda.synchronize()
        assert g.ctx.launches == n0 and still(), route
        g = GraphedStep(step, obs, warmup=2)
        want = [t.clone() for t in step(obs)]
        assert _equal(want, eager), route  # the original weights again
        assert _equal(g(obs), want), route
    # precision mode
    vima_b200.set_precision("f16f8")
    still = _sentinel(g.static_out)
    with pytest.raises(RuntimeError, match="precision mode"):
        g(obs)
    torch.cuda.synchronize()
    assert still()
    vima_b200.set_precision("f16x3")
    assert _equal(g(obs), eager)
    # without an update, many replays are what one replay is
    t0 = time.perf_counter()
    for _ in range(1000):
        out = g(obs)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    print(f"{kind}: 1000 replays in {dt * 1e3:.1f} ms, {g.weights.n_params()} parameters checked per replay")
    assert _equal(out, eager)


@pytest.mark.parametrize("kind", ["vima2M", "gato"])
def test_heads_graph_refuses_updated_weights(kind):
    """A graph over the action heads and the action embedding alone: every parameter it reads goes to the fp32 grouped GEMM
    directly, with no packed-weight cache, and it still refuses a replay after an update (and keeps the old storage alive)."""
    import vima_b200
    from vima_b200.graphs import GraphedStep

    vima_b200.set_precision("f16x3")
    pol, sd0, sd1 = _policy(kind)
    with torch.no_grad():
        pt, pm, ot, om, at = _tokens(kind, pol)
        x = _forward(kind, pol, pt, pm, ot, om, at)[-1:].clone()
    heads = torch.no_grad()(lambda inp: _heads(pol, inp))
    eager = [t.clone() for t in heads(x)]
    g = GraphedStep(heads, x, warmup=2)
    want = {id(p) for m in (pol.action_decoder, pol.action_encoder) for p in m.parameters()}
    assert want <= {id(t) for _, _, t in g.weights._slots}
    assert _equal(g(x), eager)
    for route in ("load_state_dict", "load_state_dict_assign", "new_parameter"):
        _update(pol, route, sd1)
        n0 = g.ctx.launches
        still = _sentinel(g.static_out)
        with pytest.raises(RuntimeError, match="[Cc]apture it again"):
            g(x)
        torch.cuda.synchronize()
        assert g.ctx.launches == n0 and still(), route
        new = [t.clone() for t in heads(x)]
        assert not torch.equal(new[0], eager[0]), route
        with torch.no_grad():
            for name, m, n in _parameters(pol):
                getattr(m, n).copy_(sd0[name].cuda())
        g = GraphedStep(heads, x, warmup=2)
        assert _equal(g(x), eager), route


def _slot_inputs(kind, pol, S):
    g = torch.Generator(device="cuda").manual_seed(11)
    E = pol.embed_dim
    Lp = 9
    pt = torch.randn(Lp, S, E, device="cuda", generator=g)
    pm = torch.rand(S, Lp, device="cuda", generator=g) > 0.2
    pm[:, 0] = True
    if kind.startswith("vima"):
        Q = 6
        obs = torch.randn(2, S, Q, E, device="cuda", generator=g)
        om = torch.rand(2, S, Q, device="cuda", generator=g) > 0.2
        om[..., 0] = True
        act = torch.randn(2, S, E, device="cuda", generator=g)
        return pt, pm, (lambda t: (obs[t:t + 1], om[t:t + 1], act[t:t + 1]))
    Q = pol._obj_xf_num_queries
    obs = torch.randn(2, S, Q, E, device="cuda", generator=g)
    act = torch.randn(2, S, E, device="cuda", generator=g)
    return pt, pm, (lambda t: (obs[t:t + 1], act[t:t + 1]))


def _same_state(a, b):
    return all(torch.equal(x, y) for x, y in zip(a[0], b[0])) and a[1] == b[1]


@pytest.mark.parametrize("kind", ["vima2M", "gato"])
def test_slot_graph_refuses_updated_weights(kind):
    import vima_b200

    vima_b200.set_precision("f16x3")
    pol, sd0, sd1 = _policy(kind)
    S = 3
    pt, pm, inputs = _slot_inputs(kind, pol, S)
    with torch.no_grad():
        for route in ("load_state_dict", "load_state_dict_assign", "new_parameter"):
            pol.load_state_dict({k: v.cuda() for k, v in sd0.items()})
            cache = pol.open_slots(S, max_tokens=64)
            pol.admit(cache, list(range(S)), pt, pm)
            gs = pol.capture_step_slots(cache, *inputs(0))
            eager_cache = pol.open_slots(S, max_tokens=64)
            pol.admit(eager_cache, list(range(S)), pt, pm)
            want = pol.step_slots(eager_cache, *inputs(0))
            assert torch.equal(gs(*inputs(0)), want)
            torch.cuda.synchronize()
            st = cache.state()
            _update(pol, route, sd1)
            n0 = gs.ctx.launches
            still = _sentinel([gs.static_out])
            with pytest.raises(RuntimeError, match="[Cc]apture it again"):
                gs(*inputs(1))
            torch.cuda.synchronize()
            assert gs.ctx.launches == n0 and still() and _same_state(st, cache.state()), route
            for name, m, n in _parameters(pol):
                getattr(m, n).copy_(sd0[name].cuda())
            with pytest.raises(RuntimeError, match="[Cc]apture it again"):
                gs(*inputs(1))
            assert _same_state(st, cache.state())
            with pytest.raises(ValueError, match="weights changed"):  # the cache's K/V rows belong to the weights at open
                pol.capture_step_slots(cache, *inputs(1))
        # precision mode: refused by the cache, as before
        cache = pol.open_slots(S, max_tokens=64)
        pol.admit(cache, list(range(S)), pt, pm)
        gs = pol.capture_step_slots(cache, *inputs(0))
        vima_b200.set_precision("f16f8")
        with pytest.raises(ValueError, match="precision mode"):
            gs(*inputs(0))


# ------------------------------------------------------------------------------------------------------------------------------
# 1d. decode caches
def _fstep(kind, pol, cache, t, obs, om, act):
    a = None if t == 0 else act[t - 1:t]
    if kind.startswith("vima"):
        return pol.forward_step(cache, obs[t:t + 1], om[t:t + 1], a)
    return pol.forward_step(cache, obs[t:t + 1], a)


def _sstep(kind, pol, cache, t, obs, om, act):
    a = act[t:t + 1] if t == 0 else act[t - 1:t]
    if kind.startswith("vima"):
        return pol.step_slots(cache, obs[t:t + 1], om[t:t + 1], a)
    return pol.step_slots(cache, obs[t:t + 1], a)


@pytest.mark.parametrize("kind", ["vima2M", "gato", "flamingo"])
def test_decode_caches_refuse_updated_weights(kind):
    import vima_b200

    vima_b200.set_precision("f16x3")
    pol, sd0, sd1 = _policy(kind)
    with torch.no_grad():
        pt, pm, ot, om, at = _tokens(kind, pol)
        B, T = min(2, pt.shape[1]), min(3, ot.shape[0])
        pt, pm, ot, at = pt[:, :B].contiguous(), pm[:B].contiguous(), ot[:, :B].contiguous(), at[:, :B].contiguous()
        om = None if om is None else om[:, :B].contiguous()
        dc = pol.start_decode(pt, pm, max_tokens=128)
        sc = pol.open_slots(B, max_tokens=128)
        pol.admit(sc, list(range(B)), pt, pm)
        _fstep(kind, pol, dc, 0, ot, om, at)
        _sstep(kind, pol, sc, 0, ot, om, at)
        torch.cuda.synchronize()
        _update(pol, "load_state_dict", sd1)
        L0, nv0 = dc.L, dc.n_valid.clone()
        st, mask = sc.state(), sc.mask.clone()
        pmask = None if sc.prompt_mask is None else sc.prompt_mask.clone()
        t = 1 if T > 1 else 0
        with pytest.raises(ValueError, match="weights changed"):
            _fstep(kind, pol, dc, t, ot, om, at)
        assert dc.L == L0 and torch.equal(dc.n_valid, nv0)
        for call in (lambda: _sstep(kind, pol, sc, t, ot, om, at), lambda: pol.admit(sc, [0], pt[:, :1], pm[:1])):
            with pytest.raises(ValueError, match="weights changed"):
                call()
            torch.cuda.synchronize()
            assert _same_state(st, sc.state()) and torch.equal(mask, sc.mask)
            assert pmask is None or torch.equal(pmask, sc.prompt_mask)
        # caches opened after the update follow the new weights: the full re-forward, and lockstep slots bit for bit
        dc = pol.start_decode(pt, pm, max_tokens=128)
        sc = pol.open_slots(B, max_tokens=128)
        pol.admit(sc, list(range(B)), pt, pm)
        for t in range(T):
            step = _fstep(kind, pol, dc, t, ot, om, at)
            slot = _sstep(kind, pol, sc, t, ot, om, at)
            full = _forward(kind, pol, pt, pm, ot[:t + 1], None if om is None else om[:t + 1], at)[-1:]
            assert rel_l2(full.cpu(), step.cpu()) < 2e-6, t
            assert torch.equal(step, slot), t
