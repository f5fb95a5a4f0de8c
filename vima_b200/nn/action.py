"""Action heads: ActionDecoder (12 independent 3-layer ReLU MLPs -> 700 logits -> per-head argmax) and
ActionEmbedding (4 small MLPs -> concat -> Linear).

Module surface / state-dict keys of /root/reference/vima/nn/action_decoder/{action_decoder.py:12-166, dists.py:12-28}
and action_embd/action_embd.py:9-56.  All 36 + 9 tiny GEMMs run as three (decoder) / three (embedding) grouped
exact-fp32 launches; log-softmax normalisation and the first-argmax mode run in one warp-per-head kernel.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional

import torch
import torch.nn as nn

from .. import _C
from .. import engine as eng
from .basic import F32GroupRunner, build_mlp


# ------------------------------------------------------------------------------------------------------------
# distributions (dists.py)
# ------------------------------------------------------------------------------------------------------------
class Categorical(torch.distributions.Categorical):
    def mode(self):
        return self.logits.argmax(dim=-1)


class _LazyCategorical:
    """One head of a MultiCategorical: `.logits` are the kernel-normalised log-probabilities."""

    def __init__(self, logits_norm: torch.Tensor, mode: torch.Tensor):
        self.logits = logits_norm
        self._mode = mode

    @property
    def probs(self):
        return torch.exp(self.logits)

    def mode(self):
        return self._mode

    def as_torch(self) -> Categorical:
        return Categorical(logits=self.logits)

    def sample(self, *a, **k):
        return self.as_torch().sample(*a, **k)

    def log_prob(self, v):
        return self.as_torch().log_prob(v)

    def entropy(self):
        return self.as_torch().entropy()


class MultiCategorical:
    """dists.py:12-28.  Built from raw logits (..., sum(action_dims)); normalisation + modes come from the
    `head_select` kernel (dists.py:20-28: Categorical(logits) subtracts logsumexp; mode = argmax of probs).

    `sample`, `log_prob` and `entropy` run the action-head kernel on the raw logits, kept as `raw_logits`.  Each returns one value
    per sub-head, (..., n_sub_heads); the sub-heads are independent, so the value of the joint action is the sum over the last
    dimension."""

    def __init__(self, logits: torch.Tensor = None, action_dims: List[int] = None, *, _norm=None, _modes=None):
        self._action_dims = tuple(action_dims)
        if _norm is None:
            assert logits.dim() >= 2, logits.shape
            assert logits.size(-1) == sum(self._action_dims), f"sum of action dims {self._action_dims} != {logits.size(-1)}"
            _norm, _modes = select_heads(logits, list(self._action_dims))
        self.raw_logits = logits
        self._norm, self._modes = _norm, _modes
        offs, o = [], 0
        for n in self._action_dims:
            offs.append((o, o + n))
            o += n
        self._dists = [_LazyCategorical(_norm[..., a:b], _modes[..., i]) for i, (a, b) in enumerate(offs)]

    def mode(self):
        return self._modes

    def sample(self, sampler: "ActionSampler") -> torch.Tensor:
        """One draw per sub-head from softmax(logits) at temperature 1 (the semantics of Categorical(logits=...).sample()) from
        `sampler`'s stream: int64 (..., n_sub_heads), laid out as `mode()`.  Advances the sampler by one draw."""
        return sample_heads(self.raw_logits, self._action_dims, sampler=sampler)[0]

    def log_prob(self, actions: torch.Tensor) -> torch.Tensor:
        """Log-probability of the integer `actions` (..., n_sub_heads) under each sub-head: fp32 (..., n_sub_heads), NaN where an
        index lies outside its sub-head."""
        return sample_heads(self.raw_logits, self._action_dims, actions=actions, log_prob=True)[1]

    def entropy(self) -> torch.Tensor:
        """-sum p log p of each sub-head over its p > 0 terms: fp32 (..., n_sub_heads)."""
        return sample_heads(self.raw_logits, self._action_dims, entropy=True)[2]


class ActionSampler:
    """The random stream of `MultiCategorical.sample` and of the policies' `act_slots`: a 64-bit seed and a draw counter in device
    memory.  Draw n of a sampling launch uses Philox4x32-10 with key = seed and counter = (row, sub-head, n), and the launch itself
    advances the counter on the device.  So CUDA-graph replays draw fresh numbers, and an eager run and a replayed run from the same
    seed draw the same sequence.  One sampler serves one device and one stream at a time: launches on two streams would race for
    the counter."""

    def __init__(self, seed: int, device):
        self.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
        self.counter = torch.zeros(1, dtype=torch.int64, device=device)  # the uint64 draw index

    @property
    def draws(self) -> int:
        """Sampling calls so far (one over no rows counts too).  Reads the device, so it synchronises: meant for tests."""
        return int(self.counter.item())


_head_off_cache: Dict[tuple, torch.Tensor] = {}


def _head_off(dims, device) -> torch.Tensor:
    key = (tuple(dims), str(device))
    if key not in _head_off_cache:
        off = [0]
        for n in dims:
            off.append(off[-1] + n)
        _head_off_cache[key] = torch.tensor(off, dtype=torch.int32).to(device)
    return _head_off_cache[key]


def select_heads(logits: torch.Tensor, dims: List[int]):
    """raw logits (..., sum(dims)) fp32 -> (log-softmax normalised logits, int64 modes (..., len(dims)))."""
    ctx = eng.ctx_for(logits)
    lead = logits.shape[:-1]
    total = sum(dims)
    x = logits.reshape(-1, total).float().contiguous()
    norm = torch.empty_like(x)
    modes = torch.empty((x.shape[0], len(dims)), dtype=torch.int64, device=x.device)
    ctx.head_select(x, x.shape[0], len(dims), _head_off(dims, x.device), norm, modes)
    return norm.view(*lead, total), modes.view(*lead, len(dims))


def sample_heads(logits: torch.Tensor, dims, *, sampler: Optional[ActionSampler] = None, actions: Optional[torch.Tensor] = None,
                 log_prob: bool = False, entropy: bool = False):
    """One launch of the action-head kernel on raw logits (..., sum(dims)) -> (actions, log_prob, entropy), each (..., len(dims))
    or None.  The actions are `actions` when given (scored; returned as None), else a draw from `sampler`, else the modes."""
    ctx = eng.ctx_for(logits)
    lead = logits.shape[:-1]
    n = len(dims)
    x = logits.reshape(-1, sum(dims)).float().contiguous()
    B, dev = x.shape[0], x.device
    a_in = a_out = None
    if actions is not None:
        if tuple(actions.shape) != tuple(lead) + (n,):
            raise ValueError(f"actions of shape {tuple(actions.shape)} for logits {tuple(logits.shape)} of {n} sub-heads")
        a_in = actions.to(device=dev, dtype=torch.int64).reshape(B, n).contiguous()
    else:
        a_out = torch.empty((B, n), dtype=torch.int64, device=dev)
    if sampler is not None and sampler.counter.device != dev:
        raise ValueError(f"the sampler lives on {sampler.counter.device}, the logits on {dev}")
    lp = torch.empty((B, n), dtype=torch.float32, device=dev) if log_prob else None
    ent = torch.empty((B, n), dtype=torch.float32, device=dev) if entropy else None
    ctx.head_sample(x, B, n, _head_off(dims, dev), actions_in=a_in, greedy=sampler is None,
                    seed=0 if sampler is None else sampler.seed, counter=None if sampler is None else sampler.counter,
                    actions_out=a_out, log_prob=lp, entropy=ent)
    return tuple(None if t is None else t.view(*lead, n) for t in (a_out, lp, ent))


class CategoricalHead(nn.Module):
    def forward(self, x: torch.Tensor):
        return MultiCategorical(x, [x.shape[-1]])._dists[0]


class MultiCategoricalHead(nn.Module):
    def __init__(self, action_dims: List[int]):
        super().__init__()
        self._action_dims = tuple(action_dims)

    def forward(self, x: torch.Tensor) -> MultiCategorical:
        return MultiCategorical(logits=x, action_dims=self._action_dims)


def _build_mlp_distribution_net(input_dim, *, output_dim, hidden_dim, hidden_depth, activation="relu", norm_type=None, last_layer_gain=0.01):
    mlp = build_mlp(input_dim=input_dim, output_dim=output_dim, hidden_dim=hidden_dim, hidden_depth=hidden_depth, activation=activation,
                    weight_init="orthogonal", bias_init="zeros", norm_type=norm_type)
    if last_layer_gain:
        assert last_layer_gain > 0
        nn.init.orthogonal_(mlp[-1].weight, gain=last_layer_gain)
    return mlp


class _GroupedMLPs:
    """Runs n structurally identical MLPs (same input) as one grouped exact-fp32 launch per layer."""

    def __init__(self):
        self._runners: Dict[int, List[F32GroupRunner]] = {}
        self._bufs: Dict[tuple, dict] = {}

    def run(self, mlps: List[nn.Sequential], x2: torch.Tensor, out: torch.Tensor, out_offsets: List[int]):
        ctx = eng.ctx_for(x2)
        M = x2.shape[0]
        lins = [[m for m in mlp if isinstance(m, nn.Linear)] for mlp in mlps]
        depth = len(lins[0])
        key = (M, str(x2.device), x2.shape[1])
        st = self._bufs.get(key)
        if st is None:
            st = {"x": torch.empty_like(x2), "h": []}
            for li in range(depth - 1):
                widths = [l[li].out_features for l in lins]
                st["h"].append((torch.empty((M, sum(widths)), dtype=torch.float32, device=x2.device), widths))
            st["runners"] = [F32GroupRunner() for _ in range(depth)]
            self._bufs = {key: st}  # keep one shape resident
        st["x"].copy_(x2)
        for li in range(depth):
            groups = []
            for gi, l in enumerate(lins):
                lin = l[li]
                if li == 0:
                    xin, ldx = st["x"], st["x"].stride(0)
                else:
                    hb, widths = st["h"][li - 1]
                    xin, ldx = hb[:, sum(widths[:gi]):], hb.stride(0)
                if li == depth - 1:
                    y, ldy = out[:, out_offsets[gi]:], out.stride(0)
                else:
                    hb, widths = st["h"][li]
                    y, ldy = hb[:, sum(widths[:gi]):], hb.stride(0)
                groups.append((xin, ldx, lin.weight.detach(), lin.bias.detach(), y, ldy, lin.out_features, lin.in_features))
            st["runners"][li].run(ctx, groups, M, _C.ACT_NONE if li == depth - 1 else _C.ACT_RELU)


class CategoricalNet(nn.Module):
    def __init__(self, input_dim, *, action_dim, hidden_dim, hidden_depth, activation="relu", norm_type=None, last_layer_gain=0.01):
        super().__init__()
        self.mlp = _build_mlp_distribution_net(input_dim, output_dim=action_dim, hidden_dim=hidden_dim, hidden_depth=hidden_depth,
                                               activation=activation, norm_type=norm_type, last_layer_gain=last_layer_gain)
        self.head = CategoricalHead()
        self._dims = [action_dim]

    def mlps_and_dims(self):
        return [self.mlp], self._dims

    def forward(self, x):
        eng.uses(self)  # fp32 parameters read by the kernels directly
        return ActionDecoder.run_heads([self], x)[0]


class MultiCategoricalNet(nn.Module):
    def __init__(self, input_dim, *, action_dims, hidden_dim, hidden_depth, activation="relu", norm_type=None, last_layer_gain=0.01):
        super().__init__()
        self.mlps = nn.ModuleList([
            _build_mlp_distribution_net(input_dim, output_dim=a, hidden_dim=hidden_dim, hidden_depth=hidden_depth, activation=activation,
                                        norm_type=norm_type, last_layer_gain=last_layer_gain) for a in action_dims])
        self.head = MultiCategoricalHead(action_dims)
        self._dims = list(action_dims)

    def mlps_and_dims(self):
        return list(self.mlps), self._dims

    def forward(self, x):
        eng.uses(self)  # fp32 parameters read by the kernels directly
        return ActionDecoder.run_heads([self], x)[0]


class ActionDecoder(nn.Module):
    def __init__(self, input_dim: int, *, action_dims: Dict[str, object], hidden_dim: int, hidden_depth: int, activation="relu",
                 norm_type=None, last_layer_gain: Optional[float] = 0.01):
        super().__init__()
        self._decoders = nn.ModuleDict()
        for k, v in action_dims.items():
            if isinstance(v, int):
                self._decoders[k] = CategoricalNet(input_dim, action_dim=v, hidden_dim=hidden_dim, hidden_depth=hidden_depth, activation=activation,
                                                   norm_type=norm_type, last_layer_gain=last_layer_gain)
            elif isinstance(v, list):
                self._decoders[k] = MultiCategoricalNet(input_dim, action_dims=v, hidden_dim=hidden_dim, hidden_depth=hidden_depth,
                                                        activation=activation, norm_type=norm_type, last_layer_gain=last_layer_gain)
            else:
                raise ValueError(f"Invalid action_dims value: {v}")

    _grouped = _GroupedMLPs()

    @staticmethod
    def head_logits(nets: List[nn.Module], x: torch.Tensor, grouped: Optional[_GroupedMLPs] = None):
        """All heads of all nets in three grouped launches: (raw logits fp32 [rows, sum(dims)], dims, per net its (first, end) sub-head)."""
        grouped = grouped or ActionDecoder._grouped
        x2 = x.reshape(-1, x.shape[-1]).float().contiguous()
        mlps, dims, spans = [], [], []
        for n in nets:
            m, d = n.mlps_and_dims()
            spans.append((len(dims), len(dims) + len(d)))
            mlps += m
            dims += d
        offs = [0]
        for n_ in dims:
            offs.append(offs[-1] + n_)
        logits = torch.empty((x2.shape[0], offs[-1]), dtype=torch.float32, device=x.device)
        grouped.run(mlps, x2, logits, offs[:-1])
        return logits, dims, spans

    @staticmethod
    def run_heads(nets: List[nn.Module], x: torch.Tensor, grouped: Optional[_GroupedMLPs] = None):
        """All heads of all nets in three grouped launches + one head_select launch; returns one dist per net."""
        lead = x.shape[:-1]
        logits, dims, spans = ActionDecoder.head_logits(nets, x, grouped)
        offs = [0]
        for n_ in dims:
            offs.append(offs[-1] + n_)
        norm, modes = select_heads(logits.view(*lead, offs[-1]), dims)
        out = []
        for net, (a, b) in zip(nets, spans):
            mc = MultiCategorical(action_dims=dims[a:b], _norm=norm[..., offs[a]:offs[b]], _modes=modes[..., a:b])
            mc.raw_logits = logits.view(*lead, offs[-1])[..., offs[a]:offs[b]]
            out.append(mc._dists[0] if isinstance(net, CategoricalNet) else mc)
        return out

    def forward(self, x: torch.Tensor):
        """(..., E) -> {key: MultiCategorical}  (action_decoder.py:51-52)."""
        eng.uses(self)  # fp32 parameters read by the kernels directly
        if not hasattr(self, "_my_grouped"):
            self._my_grouped = _GroupedMLPs()
        keys = list(self._decoders.keys())
        dists = ActionDecoder.run_heads([self._decoders[k] for k in keys], x, self._my_grouped)
        return dict(zip(keys, dists))


# ------------------------------------------------------------------------------------------------------------
# action embedding (action_embd.py)
# ------------------------------------------------------------------------------------------------------------
class ContinuousActionEmbedding(nn.Module):
    def __init__(self, output_dim: int, *, input_dim: int, hidden_dim: int, hidden_depth: int):
        super().__init__()
        self._layer = build_mlp(input_dim=input_dim, hidden_dim=hidden_dim, output_dim=output_dim, hidden_depth=hidden_depth)
        self.output_dim = output_dim

    def forward(self, x: torch.Tensor):
        eng.uses(self)  # fp32 parameters read by the kernels directly
        if not hasattr(self, "_g"):
            self._g = _GroupedMLPs()
        lead = x.shape[:-1]
        x2 = x.reshape(-1, x.shape[-1]).float().contiguous()
        out = torch.empty((x2.shape[0], self.output_dim), dtype=torch.float32, device=x.device)
        self._g.run([self._layer], x2, out, [0])
        return out.view(*lead, self.output_dim)


class ActionEmbedding(nn.Module):
    def __init__(self, output_dim: int, *, embed_dict: Dict[str, nn.Module]):
        super().__init__()
        self._embed_dict = nn.ModuleDict(embed_dict)
        embed_dict_output_dim = sum(embed_dict[k].output_dim for k in sorted(embed_dict.keys()))
        self._post_layer = nn.Identity() if output_dim == embed_dict_output_dim else nn.Linear(embed_dict_output_dim, output_dim)
        self._output_dim = output_dim
        self._input_fields_checked = False
        self._runners = {}

    @property
    def output_dim(self):
        return self._output_dim

    def forward(self, x_dict: Dict[str, torch.Tensor]):
        """{key: (..., n_k) float} -> (..., output_dim): per-key MLP, concat in SORTED key order, Linear (:29-37)."""
        eng.uses(self)  # fp32 parameters read by the kernels directly
        if not self._input_fields_checked:
            assert set(x_dict.keys()) == set(self._embed_dict.keys())
            self._input_fields_checked = True
        keys = sorted(x_dict.keys())
        x0 = x_dict[keys[0]]
        ctx = eng.ctx_for(x0)
        lead = x0.shape[:-1]
        dev = x0.device
        M = 1
        for s in lead:
            M *= s
        widths = [self._embed_dict[k].output_dim for k in keys]
        cat = torch.empty((M, sum(widths)), dtype=torch.float32, device=dev)
        # layer-wise grouped launches over the 4 embedders (they are structurally identical 2-layer MLPs)
        lins = [[m for m in self._embed_dict[k]._layer if isinstance(m, nn.Linear)] for k in keys]
        depth = len(lins[0])
        assert all(len(l) == depth for l in lins)
        st = self._runners.setdefault((M, str(dev)), {"r": [F32GroupRunner() for _ in range(depth + 1)], "bufs": {}})
        cur = [x_dict[k].reshape(M, -1).float().contiguous() for k in keys]
        for li in range(depth):
            last = li == depth - 1
            groups, nxt = [], []
            for gi, (k, l) in enumerate(zip(keys, lins)):
                lin = l[li]
                if last:
                    y = cat[:, sum(widths[:gi]):]
                    ldy = cat.stride(0)
                else:
                    buf = st["bufs"].setdefault((li, gi), torch.empty((M, lin.out_features), dtype=torch.float32, device=dev))
                    y, ldy = buf, buf.stride(0)
                xin = cur[gi]
                if li == 0:  # inputs come from the caller: stage them in resident buffers so descriptors stay valid
                    xb = st["bufs"].setdefault(("x", gi), torch.empty_like(xin))
                    xb.copy_(xin)
                    xin = xb
                groups.append((xin, xin.stride(0), lin.weight.detach(), lin.bias.detach(), y, ldy, lin.out_features, lin.in_features))
                nxt.append(y)
            st["r"][li].run(ctx, groups, M, _C.ACT_NONE if last else _C.ACT_RELU)
            cur = nxt
        if isinstance(self._post_layer, nn.Identity):
            return cat.view(*lead, -1)
        out = torch.empty((M, self._output_dim), dtype=torch.float32, device=dev)
        pl = self._post_layer
        st["r"][depth].run(ctx, [(cat, cat.stride(0), pl.weight.detach(), pl.bias.detach(), out, out.stride(0), pl.out_features, pl.in_features)], M, _C.ACT_NONE)
        return out.view(*lead, self._output_dim)
