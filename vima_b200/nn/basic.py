"""Leaf modules: parameter holders with the reference's state-dict keys whose `forward` runs on the C-ABI kernels.

Mirrors /root/reference/vima/nn/utils.py (`Embedding` :9-12, `build_mlp` :15-111) and the HF `Conv1D`
(HF:pytorch_utils.py:97-123) the reference's decoder uses for c_attn / c_fc / c_proj.
"""
from __future__ import annotations

import ctypes as C
from typing import Callable, List, Optional

import torch
import torch.nn as nn

from .. import _C
from .. import engine as eng


class Embedding(nn.Embedding):
    """vima/nn/utils.py:9-12 (index gather only; the policy fuses the lookups it needs into its own kernels)."""

    @property
    def output_dim(self):
        return self.embedding_dim


class Conv1D(nn.Module):
    """HF Conv1D parameter holder: weight [in, out], bias [out] (y = x @ W + b)."""

    def __init__(self, nf: int, nx: int):
        super().__init__()
        self.nf = nf
        self.weight = nn.Parameter(torch.empty(nx, nf).normal_(std=0.02))
        self.bias = nn.Parameter(torch.zeros(nf))


# ------------------------------------------------------------------------------------------------------------
# exact-fp32 grouped GEMM helper (CUDA cores) for the tiny layers
# ------------------------------------------------------------------------------------------------------------
class F32GroupRunner:
    """One grouped fp32 GEMM launch.  The descriptors are built on the host and travel in the kernel's parameter space
    (`vima_gemm_f32_grouped_host`): no device-side array, no host->device copy, capturable into a CUDA graph."""

    def __init__(self):
        self._key = None
        self._arr = None
        self._meta = None

    def run(self, ctx: _C.Context, groups: List[tuple], M: int, act: int):
        """groups: (x, ldx, w, b|None, y, ldy, n, k) with tensors / ints; x,w,y column offsets already applied via views."""
        key = tuple((g[0].data_ptr(), g[1], g[2].data_ptr(), 0 if g[3] is None else g[3].data_ptr(), g[4].data_ptr(), g[5], g[6], g[7]) for g in groups)
        if key != self._key:
            arr = (_C.F32GemmGroup * len(groups))()
            for i, k in enumerate(key):
                arr[i] = _C.F32GemmGroup(k[0], k[1], k[2], groups[i][2].stride(0), k[3] or None, k[4], k[5], k[6], k[7])
            self._arr, self._key = arr, key
            self._meta = (len(groups), max(k[6] for k in key))
        ctx.gemm_f32_grouped_host(self._arr, self._meta[0], M, self._meta[1], act)


def _use_tensor_cores(in_features: int, rows: int) -> bool:
    # wgmma path needs K % 8 == 0 (TMA row pitch); tiny-K layers run exact fp32 on CUDA cores
    return in_features % 8 == 0 and in_features >= 64


class Linear(nn.Linear):
    """nn.Linear with the reference's parameters whose forward is the wgmma GEMM (or exact fp32 for tiny K)."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self._wc = eng.WeightCache(self)
        self._f32 = F32GroupRunner()

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        eng.uses(self)  # fp32 parameters read by the kernels directly
        ctx = eng.ctx_for(x)
        p = eng.prec()
        lead = x.shape[:-1]
        x2 = x.reshape(-1, self.in_features)
        if _use_tensor_cores(self.in_features, x2.shape[0]):
            pw = self._wc.get("w", (self.weight, self.bias), lambda: eng.pack_linear(ctx, self.weight, self.bias, transposed=False, p=p))
            out, _ = eng.gemm(ctx, eng.to_operand(ctx, x2, p), pw, p, want_f32=True)
        else:
            out = simt_linear(ctx, self._f32, x2, self.weight, self.bias, _C.ACT_NONE)
        return out.view(*lead, self.out_features)


def simt_linear(ctx, runner: F32GroupRunner, x2: torch.Tensor, weight, bias, act: int, out: Optional[torch.Tensor] = None):
    x2 = x2.float().contiguous()
    M = x2.shape[0]
    w = weight.detach()
    b = None if bias is None else bias.detach()
    if out is None:
        out = torch.empty((M, w.shape[0]), dtype=torch.float32, device=x2.device)
    if M:
        runner.run(ctx, [(x2, x2.stride(0), w, b, out, out.stride(0), w.shape[0], w.shape[1])], M, act)
    return out


class MLPSequential(nn.Sequential):
    """`build_mlp`'s nn.Sequential (Linear, Identity, ReLU, ..., Linear -> keys 0/3/6) with a fused forward:
    every hidden activation stays a 16-bit operand pair, ReLU lives in the GEMM epilogue."""

    def _linears(self):
        return [m for m in self if isinstance(m, nn.Linear)]

    def forward(self, x: torch.Tensor, *, want16: bool = False, out16_ld: Optional[int] = None, out16: Optional[eng.Opnd] = None):
        eng.uses(self)  # fp32 parameters read by the kernels directly
        ctx = eng.ctx_for(x)
        p = eng.prec()
        lins = self._linears()
        want16 = want16 or out16 is not None
        if not hasattr(self, "_wc"):
            self._wc = eng.WeightCache(self)
            self._f32 = [F32GroupRunner() for _ in lins]
        lead = x.shape[:-1]
        cur32: Optional[torch.Tensor] = x.reshape(-1, lins[0].in_features)
        cur16: Optional[eng.Opnd] = None
        rows = cur32.shape[0]
        for i, lin in enumerate(lins):
            last = i + 1 == len(lins)
            act = _C.ACT_NONE if last else _C.ACT_RELU
            if _use_tensor_cores(lin.in_features, rows):
                pw = self._wc.get(f"l{i}", (lin.weight, lin.bias), lambda lin=lin: eng.pack_linear(ctx, lin.weight, lin.bias, transposed=False, p=p))
                a = cur16 if cur16 is not None else eng.to_operand(ctx, cur32, p)
                if last:
                    cur32, cur16 = eng.gemm(ctx, a, pw, p, act=act, want_f32=not want16, want16=want16 and out16 is None, out16_ld=out16_ld, out16=out16)
                else:
                    cur32, cur16 = eng.gemm(ctx, a, pw, p, act=act, want16=True)
            else:
                src = cur32 if cur32 is not None else cur16.float(p)
                cur32, cur16 = simt_linear(ctx, self._f32[i], src, lin.weight, lin.bias, act), None
        if want16:
            if cur16 is None:
                cur16 = eng.to_operand(ctx, cur32, p)
                if out16 is not None:
                    raise NotImplementedError("out16 needs a tensor-core final layer")
            return cur16
        return cur32.view(*lead, lins[-1].out_features)


def get_activation(activation) -> Callable:
    if not activation:
        return nn.Identity
    if callable(activation):
        return activation
    table = {
        "tanh": nn.Tanh,
        "relu": lambda: nn.ReLU(inplace=True),
        "leaky_relu": lambda: nn.LeakyReLU(inplace=True),
        "swish": lambda: nn.SiLU(inplace=True),
        "sigmoid": nn.Sigmoid,
        "elu": lambda: nn.ELU(inplace=True),
        "gelu": nn.GELU,
    }
    activation = activation.lower()
    assert activation in table, f"Supported activations: {table.keys()}"
    return table[activation]


def build_mlp(
    input_dim,
    *,
    hidden_dim: int,
    output_dim: int,
    hidden_depth: int = None,
    num_layers: int = None,
    activation="relu",
    weight_init="orthogonal",
    bias_init="zeros",
    norm_type=None,
    add_input_activation=False,
    add_input_norm: bool = False,
    add_output_activation=False,
    add_output_norm: bool = False,
) -> nn.Sequential:
    """Same signature and module layout as vima/nn/utils.py:15-111.  The fused kernels cover the configuration the
    policy uses (ReLU, no norm, no input/output extras); anything else is refused rather than silently run in eager."""
    assert (hidden_depth is None) != (num_layers is None), "Either hidden_depth or num_layers must be specified, but not both."
    hidden_depth = num_layers - 1 if hidden_depth is None else hidden_depth
    assert hidden_depth >= 0
    if norm_type or add_input_activation or add_input_norm or add_output_activation or add_output_norm or (
        isinstance(activation, str) and activation.lower() != "relu"
    ) or callable(activation):
        raise NotImplementedError("vima_b200.build_mlp implements the ReLU / no-norm configuration the VIMA policy uses")
    act_layer = get_activation(activation)
    if hidden_depth == 0:
        mods = [nn.Linear(input_dim, output_dim)]
    else:
        mods = [nn.Linear(input_dim, hidden_dim), nn.Identity(), act_layer()]
        for _ in range(hidden_depth - 1):
            mods += [nn.Linear(hidden_dim, hidden_dim), nn.Identity(), act_layer()]
        mods.append(nn.Linear(hidden_dim, output_dim))
    gain = nn.init.calculate_gain("relu")
    for m in mods:
        if isinstance(m, nn.Linear):
            if weight_init == "orthogonal":
                nn.init.orthogonal_(m.weight, gain=gain)
            elif isinstance(weight_init, str):
                getattr(nn.init, f"{weight_init}_")(m.weight)
            else:
                weight_init(m.weight)
            if bias_init == "zeros":
                nn.init.zeros_(m.bias)
            elif isinstance(bias_init, str):
                getattr(nn.init, f"{bias_init}_")(m.bias)
            else:
                bias_init(m.bias)
    return MLPSequential(*mods)
