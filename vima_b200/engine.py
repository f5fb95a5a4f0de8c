"""Host-side glue between the `vima_b200.nn` modules and the C-ABI kernels: precision mode, 16-bit operand
buffers, packed-weight cache and one thin wrapper per kernel family.  torch only owns memory and streams here.

Precision modes (DESIGN.md "operand precision"):
    "f16x3"  fp16 (hi, lo) operand pairs, three-term products -> fp32-equivalent (parity mode, default)
    "bf16x3" same with bf16 pairs (fp32 dynamic range, ~16-bit significand)
    "f16"    single-pass fp16 operands (11-bit significand, TF32-class accuracy)
    "bf16"   single-pass bf16 operands (BASELINE.json configs[1])
    "f16f8"  fp16 hi*hi plus the two cross terms in e4m3 at the fp8 tensor rate for the decoder GEMMs (2 pass-equivalents
             instead of 3; ~4e-4 end to end); attention, ViT and T5 stay on the three-term fp16 products
Accumulation, softmax, LayerNorm, residuals and biases are fp32 in every mode.
"""
from __future__ import annotations

import contextlib
import math
import weakref
from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import torch

from . import _C

_MODES = {"f16x3": (_C.DT_F16, True), "bf16x3": (_C.DT_BF16, True), "f16": (_C.DT_F16, False), "bf16": (_C.DT_BF16, False),
          "f16f8": (_C.DT_F16, True)}
_precision = "f16x3"


def set_precision(mode: str) -> None:
    global _precision
    if mode not in _MODES:
        raise ValueError(f"precision must be one of {sorted(_MODES)}")
    _precision = mode


def get_precision() -> str:
    return _precision


@dataclass(frozen=True)
class Prec:
    name: str
    dtype: int
    split: bool
    f8: bool = False  # decoder GEMM operands carry e4m3 cross-term views instead of a 16-bit lo part


def prec() -> Prec:
    dt, sp = _MODES[_precision]
    return Prec(_precision, dt, sp, _precision == "f16f8")


def ctx_for(t: torch.Tensor) -> _C.Context:
    if not t.is_cuda:
        raise RuntimeError(
            "vima_b200 modules only run on a CUDA (sm_90a) device: got a CPU tensor. There is no CPU / eager fallback."
        )
    return _C.Context.get(t.device)


def round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


class Opnd:
    """A [rows, cols] activation as 16-bit GEMM operand(s): hi (and lo in split mode), leading dim `ld` (mult. of 8)."""

    __slots__ = ("hi", "lo", "rows", "cols", "ld", "lo8", "hi8")

    def __init__(self, rows: int, cols: int, device, split: bool, ld: Optional[int] = None, zero: bool = False, f8: bool = False):
        """split: 16-bit lo part; f8: e4m3 cross-term views (lo8, hi8) INSTEAD of the 16-bit lo part ("f16f8" GEMM inputs)."""
        self.rows, self.cols = rows, cols
        self.ld = round_up(cols, 8) if ld is None else ld
        mk = torch.zeros if (zero or self.ld != cols) else torch.empty
        self.hi = mk((max(rows, 1), self.ld), dtype=torch.int16, device=device)
        self.lo = mk((max(rows, 1), self.ld), dtype=torch.int16, device=device) if (split and not f8) else None
        self.lo8 = self.hi8 = None
        if f8:
            ld8 = round_up(cols, 16)
            self.lo8 = torch.zeros((max(rows, 1), ld8), dtype=torch.uint8, device=device) if ld8 != cols else torch.empty((max(rows, 1), ld8), dtype=torch.uint8, device=device)
            self.hi8 = torch.zeros_like(self.lo8) if ld8 != cols else torch.empty_like(self.lo8)

    def sub(self, r0: int, n_rows: int, c0: int = 0, n_cols: Optional[int] = None) -> "Opnd":
        """A window [r0:r0+n_rows, c0:c0+n_cols] sharing storage (as GEMM input c0 must be a multiple of 8)."""
        v = object.__new__(Opnd)
        v.rows, v.cols, v.ld = n_rows, (self.cols - c0 if n_cols is None else n_cols), self.ld
        v.hi = self.hi[r0 : r0 + max(n_rows, 1), c0:]
        v.lo = None if self.lo is None else self.lo[r0 : r0 + max(n_rows, 1), c0:]
        v.lo8 = None if self.lo8 is None else self.lo8[r0 : r0 + max(n_rows, 1), c0:]
        v.hi8 = None if self.hi8 is None else self.hi8[r0 : r0 + max(n_rows, 1), c0:]
        return v

    def float(self, p: Prec) -> torch.Tensor:
        """Debug / tests: reconstruct fp32."""
        tdt = torch.float16 if p.dtype == _C.DT_F16 else torch.bfloat16
        x = self.hi.view(tdt)[: self.rows, : self.cols].float()
        if self.lo is not None:
            x = x + self.lo.view(tdt)[: self.rows, : self.cols].float()
        return x


class PackedWeight:
    """K-major 16-bit packed weight [n_rows, ld] (+lo), optional fp32 bias in accumulator-column order."""

    __slots__ = ("hi", "lo", "n", "k", "ld", "inv_scale", "bias", "glu", "block_n", "n_out", "hi8", "lo8", "ln_c1", "ln_cols")


def _pow2_scale(w_absmax: float, p: Prec) -> float:
    if p.dtype != _C.DT_F16 or w_absmax <= 0 or not math.isfinite(w_absmax):
        return 1.0
    # max |w| * scale in [512, 1024): keeps the lo part of all but tiny weights in fp16's normal range
    return 2.0 ** math.floor(math.log2(1024.0 / w_absmax))


def fold_layernorm(w_nk: torch.Tensor, bias: Optional[torch.Tensor], gamma: torch.Tensor, beta: Optional[torch.Tensor], rows: Optional[torch.Tensor] = None):
    """LayerNorm folded into the Linear that consumes it:  W (gamma*(x-mean)*rstd + beta) + b
         = rstd * ((W*gamma) x - mean * c1) + c2,   c1 = rowsum(W*gamma),  c2 = b + W beta.
    w_nk: [n, k] fp32.  `rows`: bool [n] selecting the output rows the fold applies to (None = all; the others stay as they are).
    Returns (W', c1, c2) fp32, computed in fp64."""
    w64 = w_nk.double()
    g = gamma.detach().double()
    wp = w64 * g[None, :]
    c1 = wp.sum(dim=1)
    c2 = torch.zeros(w_nk.shape[0], dtype=torch.float64, device=w_nk.device) if bias is None else bias.detach().double().clone()
    add = torch.zeros_like(c2) if beta is None else w64 @ beta.detach().double()
    if rows is not None:
        wp = torch.where(rows[:, None], wp, w64)
        c1 = torch.where(rows, c1, torch.zeros_like(c1))
        add = torch.where(rows, add, torch.zeros_like(add))
    return wp.float().contiguous(), c1.float().contiguous(), (c2 + add).float().contiguous()


def pack_linear(ctx: _C.Context, weight: torch.Tensor, bias: Optional[torch.Tensor], *, transposed: bool, p: Prec, f8: bool = False,
                ln: Optional[Tuple[torch.Tensor, Optional[torch.Tensor]]] = None) -> PackedWeight:
    """nn.Linear weight [n, k] or HF Conv1D weight [k, n] (transposed=True).  f8: also the e4m3 cross-term views.
    ln = (gamma, beta): the LayerNorm that feeds this layer is folded into the packed weight / bias (see `fold_layernorm`); the
    GEMM then takes the UN-normalised rows plus their (mean, rstd)."""
    w = weight.detach()
    if w.dtype != torch.float32:
        w = w.float()
    ln_c1 = None
    if ln is not None:
        w_nk = w.t() if transposed else w
        w, ln_c1, bias = fold_layernorm(w_nk.contiguous(), bias, ln[0], ln[1])
        transposed = False
    w = w.contiguous()
    n, k = (w.shape[1], w.shape[0]) if transposed else (w.shape[0], w.shape[1])
    pw = PackedWeight()
    pw.n, pw.k, pw.ld = n, k, round_up(k, 8)
    scale = _pow2_scale(float(w.abs().max()), p)
    pw.inv_scale = 1.0 / scale
    pw.hi = torch.empty((n, pw.ld), dtype=torch.int16, device=w.device)
    pw.lo = torch.empty_like(pw.hi) if p.split else None
    f8 = f8 and p.f8
    pw.lo = None if f8 else pw.lo
    ctx.pack_weight(w, pw.hi, pw.lo, transposed=transposed, scale=scale, dtype=p.dtype)
    pw.hi8 = pw.lo8 = None
    if f8:
        pw.hi8 = torch.empty((n, round_up(k, 16)), dtype=torch.uint8, device=w.device)
        pw.lo8 = torch.empty_like(pw.hi8)
        ctx.pack_weight_f8(w, pw.hi8, pw.lo8, transposed=transposed, scale=scale)
    pw.bias = None if bias is None else bias.detach().float().contiguous()
    pw.glu, pw.block_n, pw.n_out = 0, 0, n
    pw.ln_c1, pw.ln_cols = ln_c1, (1 if ln_c1 is not None else 0)
    return pw


def pack_glu(ctx: _C.Context, w_val: torch.Tensor, b_val: Optional[torch.Tensor], w_gate: torch.Tensor, *, val_transposed: bool,
             gate_transposed: bool, p: Prec, f8: bool = False, ln: Optional[Tuple[torch.Tensor, Optional[torch.Tensor]]] = None,
             ln_gate: bool = True) -> PackedWeight:
    """Interleaves value / gate rows per accumulator tile so one GEMM + GLU epilogue yields act(x Wv + b) * (x Wg).
    ln = (gamma, beta): fold the LayerNorm in front of the value projection (and of the gate projection when `ln_gate`; the
    XAttention gate reads the un-normalised stream, components.py:218-221) into the packed weights."""
    wv = w_val.detach().float()
    wg = w_gate.detach().float()
    wv = wv.t() if val_transposed else wv
    wg = wg.t() if gate_transposed else wg
    n_out, k = wv.shape
    assert wg.shape == (n_out, k)
    c1v = c1g = bg = None
    if ln is not None:
        wv, c1v, b_val = fold_layernorm(wv.contiguous(), b_val, ln[0], ln[1])
        if ln_gate:
            wg, c1g, bg = fold_layernorm(wg.contiguous(), None, ln[0], ln[1])
    bn = ctx.glu_block_n(n_out)
    half = bn // 2
    tiles = (n_out + half - 1) // half
    dev = wv.device
    W = torch.zeros((tiles, 2, half, k), dtype=torch.float32, device=dev)
    Bv = torch.zeros((tiles, 2, half), dtype=torch.float32, device=dev)
    pad = tiles * half - n_out
    wv_p = torch.nn.functional.pad(wv, (0, 0, 0, pad)).view(tiles, half, k)
    wg_p = torch.nn.functional.pad(wg, (0, 0, 0, pad)).view(tiles, half, k)
    W[:, 0] = wv_p
    W[:, 1] = wg_p
    if b_val is not None:
        Bv[:, 0] = torch.nn.functional.pad(b_val.detach().float(), (0, pad)).view(tiles, half)
    if bg is not None:
        Bv[:, 1] = torch.nn.functional.pad(bg, (0, pad)).view(tiles, half)
    pw = pack_linear(ctx, W.view(tiles * bn, k), Bv.view(tiles * bn), transposed=False, p=p, f8=f8)
    pw.glu, pw.block_n, pw.n_out = 1, bn, n_out
    if ln is not None:
        C1 = torch.zeros((tiles, 2, half), dtype=torch.float32, device=dev)
        C1[:, 0] = torch.nn.functional.pad(c1v, (0, pad)).view(tiles, half)
        if c1g is not None:
            C1[:, 1] = torch.nn.functional.pad(c1g, (0, pad)).view(tiles, half)
        pw.ln_c1, pw.ln_cols = C1.view(tiles * bn).contiguous(), (1 if ln_gate else 2)
    return pw


# -------------------------------------------------------------------------------------------------------------
# packed-weight cache: keyed by the parameters' identity + in-place version, the device and the precision mode
# -------------------------------------------------------------------------------------------------------------
class WeightCache:
    """Packed weights of one module (`owner`).  An entry is rebuilt when a parameter it was packed from is replaced (new storage:
    `load_state_dict(assign=True)`, `module.weight = nn.Parameter(...)`, `param.data = t`), written in place through autograd
    (`load_state_dict`, `copy_` / `mul_` under no_grad: the version counter moves), moved to another device, or when the precision
    mode changes.  A write through `param.data` (`param.data.copy_(t)`) moves no version counter and is not seen: call
    `refresh_weights(module)` after one.  `generation` counts the clears, so a captured graph or an open decode cache can tell."""

    def __init__(self, owner: Optional[torch.nn.Module] = None):
        self._store: Dict[str, Tuple[tuple, object]] = {}
        self._owner = None if owner is None else weakref.ref(owner)  # weak: no module <-> cache reference cycle
        self.generation = 0

    @property
    def owner(self) -> Optional[torch.nn.Module]:
        return None if self._owner is None else self._owner()

    def get(self, name: str, params: Tuple[Optional[torch.Tensor], ...], build):
        p = prec()
        key = (p.name,) + tuple((None if t is None else (t.data_ptr(), t._version, str(t.device))) for t in params)
        hit = self._store.get(name)
        # the entry also holds weak references to the tensors it was packed from: a replacement that lands in the block its
        # predecessor freed (same address, same version) is still another tensor
        if hit is not None and hit[0] == key and all((r is None) if t is None else (r is not None and r() is t) for r, t in zip(hit[2], params)):
            val = hit[1]
        else:
            val = build()
            self._store[name] = (key, val, tuple(None if t is None else weakref.ref(t) for t in params))
        if _recorders:
            _recorders[-1].note(self, params, val)
        return val

    def clear(self):
        self._store.clear()
        self.generation += 1

    def __deepcopy__(self, memo):  # a copied module gets an empty cache owned by the copy
        owner = self.owner
        return WeightCache(None if owner is None else memo.get(id(owner), owner))

    def __getstate__(self):  # packed weights and the owner link are not pickled; the unpickled module repacks
        return {}

    def __setstate__(self, state):
        self.__init__()


def refresh_weights(module: torch.nn.Module) -> None:
    """Drop every packed weight under `module`; the next call repacks from the parameters as they are.  Needed after a write through
    `param.data` (which moves no version counter, see WeightCache); graphs captured and decode caches opened before it refuse to run."""
    for m in module.modules():
        wc = m.__dict__.get("_wc")
        if isinstance(wc, WeightCache):
            wc.clear()


def uses(module: torch.nn.Module) -> None:
    """Called where a module's fp32 parameters go to a kernel without a packed-weight cache (the fp32 grouped GEMMs of the action
    heads and embeddings, embedding tables, norm gains): while a graph is being captured (`record_weights`), the module becomes one
    the graph depends on, as the owner of a cache the step used does."""
    if _recorders:
        _recorders[-1].note_module(module)


class WeightState:
    """What a captured graph or an open decode cache depends on: the identity, storage and in-place version of every parameter
    under `modules`, of the (module, name) parameters in `slots` (plus `params` of caches without an owner module) and the clear count of every packed-weight cache there.  It keeps references to those parameters (and to `keep`, the packed
    weights a graph read), so nothing the device pointers point at is freed while it lives."""

    def __init__(self, modules=(), params=(), keep=(), slots=()):
        self.precision = prec().name
        self._slots, self._caches, seen, seen_c = [], [], set(), set()
        for root in modules:
            for m in root.modules():
                wc = m.__dict__.get("_wc")
                if isinstance(wc, WeightCache) and id(wc) not in seen_c:
                    seen_c.add(id(wc))
                    self._caches.append(wc)
                for n, t in m._parameters.items():
                    if t is not None and (id(m._parameters), n) not in seen:
                        seen.add((id(m._parameters), n))
                        self._slots.append((m._parameters, n, t))
        for m, n in slots:
            if (id(m._parameters), n) not in seen:
                seen.add((id(m._parameters), n))
                self._slots.append((m._parameters, n, m._parameters[n]))
        self._loose = tuple(t for t in params if t is not None)
        self._keep = list(keep)
        self._fp = self._current()

    def _current(self) -> tuple:
        return (tuple(c.generation for c in self._caches),
                tuple((t.data_ptr(), t._version) if d.get(n) is t else None for d, n, t in self._slots),
                tuple((t.data_ptr(), t._version) for t in self._loose))

    def n_params(self) -> int:
        return len(self._slots) + len(self._loose)

    def changed(self) -> Optional[str]:
        """None while every parameter and cache recorded is as it was; otherwise what moved.  (The precision mode is checked by the
        caller: `precision` holds the one in force when this was taken.)"""
        if self._current() != self._fp:
            return "the weights changed (a parameter was replaced, written in place, or refresh_weights was called)"
        return None

    def matches(self, other: "WeightState") -> bool:
        """Both were taken of the same parameters and packed-weight caches at the same versions, and neither has changed since."""
        return self._fp == other._fp and self.changed() is None and other.changed() is None


class _Recorder:
    def __init__(self):
        self.owners, self.params, self.values, self._seen = [], [], [], set()

    def note_module(self, module: torch.nn.Module) -> None:
        if id(module) not in self._seen:
            self._seen.add(id(module))
            self.owners.append(module)

    def note(self, cache: WeightCache, params, val) -> None:
        self.values.append(val)
        owner = cache.owner
        if owner is not None:
            self.note_module(owner)
        elif id(cache) not in self._seen:
            self._seen.add(id(cache))
            self.params.extend(params)


@contextlib.contextmanager
def record_weights():
    """Collects every packed-weight cache used inside the block and every module passed to `uses`; yields a callable returning the
    WeightState of those modules (all their parameters) holding the packed weights used."""
    rec = _Recorder()
    _recorders.append(rec)
    try:
        yield lambda: WeightState(rec.owners, rec.params, rec.values)
    finally:
        _recorders.remove(rec)


_recorders: list = []


# -------------------------------------------------------------------------------------------------------------
# op wrappers
# -------------------------------------------------------------------------------------------------------------
def gemm(ctx: _C.Context, a: Opnd, w: PackedWeight, p: Prec, *, act=_C.ACT_NONE, residual=None, mul=None, out_f32: Optional[torch.Tensor] = None,
         out16: Optional[Opnd] = None, want_f32=False, want16=False, out16_ld: Optional[int] = None, rows: Optional[int] = None,
         out_f8: bool = False, row_stats: Optional[torch.Tensor] = None, res_ln=None, stats_out: Optional[torch.Tensor] = None):
    """out = epilogue(a @ w^T).  Returns (out_f32 | None, out16 | None).  out_f8: the 16-bit output carries e4m3 cross-term views
    (it feeds an "f16f8" GEMM) instead of a 16-bit lo part (attention inputs keep the 16-bit pair).
    row_stats: fp32 [M, 2] (mean, rstd) of the rows of `a` for a weight packed with a folded LayerNorm (`pack_*(ln=...)`).
    res_ln = (stats [M,2], gamma, beta): the residual rows are LayerNorm'd on the fly.  stats_out: fp32 [M, parts, 2] receiving the
    per-row partial (sum, sum of squares) of the output (`stats_buffer`, `row_stats_of`)."""
    M = a.rows if rows is None else rows
    if a.cols != w.k:
        raise ValueError(f"gemm: operand has {a.cols} columns, weight expects {w.k}")
    dev = a.hi.device
    if want_f32 and out_f32 is None:
        out_f32 = torch.empty((M, w.n_out), dtype=torch.float32, device=dev)
    if want16 and out16 is None:
        out16 = Opnd(M, w.n_out, dev, p.split, ld=out16_ld, f8=out_f8 and p.f8)
    if (row_stats is None) != (w.ln_c1 is None):
        raise RuntimeError("gemm: a weight packed with a folded LayerNorm needs the operand's row statistics (and only such a weight takes them)")
    if M == 0:
        return out_f32, out16
    use_f8 = a.lo8 is not None and w.lo8 is not None
    if not use_f8 and p.split and (a.lo is None or w.lo is None):
        raise RuntimeError("gemm: operand formats do not match (16-bit lo part missing on one side)")
    ctx.gemm(M=M, N=w.n, K=w.k, a_hi=a.hi, a_lo=None if use_f8 else a.lo, lda=a.ld, b_hi=w.hi, b_lo=None if use_f8 else w.lo, ldb=w.ld,
             dtype=p.dtype, glu=w.glu, act=act, acc_scale=w.inv_scale, bias=w.bias, mul=mul, residual=residual, out_f32=out_f32,
             out_hi=None if out16 is None else out16.hi, out_lo=None if out16 is None else out16.lo,
             ld_o16=0 if out16 is None else out16.ld, block_n=w.block_n,
             a_lo8=a.lo8 if use_f8 else None, a_hi8=a.hi8 if use_f8 else None, b_hi8=w.hi8 if use_f8 else None, b_lo8=w.lo8 if use_f8 else None,
             out_lo8=None if out16 is None else out16.lo8, out_hi8=None if out16 is None else out16.hi8,
             row_stats=row_stats, ln_c1=w.ln_c1, ln_cols=w.ln_cols if row_stats is not None else 0,
             res_stats=None if res_ln is None else res_ln[0], res_gamma=None if res_ln is None else res_ln[1],
             res_beta=None if res_ln is None else res_ln[2], stats_out=stats_out)
    return out_f32, out16


def stats_buffer(ctx: _C.Context, M: int, w: PackedWeight, device) -> torch.Tensor:
    """fp32 [M, parts, 2] for the partial row statistics a GEMM with weight `w` emits."""
    return torch.empty((max(M, 1), ctx.gemm_stats_parts(w.n, w.glu, w.block_n), 2), dtype=torch.float32, device=device)


def row_stats_of(ctx: _C.Context, partial: torch.Tensor, rows: int, cols: int, eps: float, rms: bool = False) -> torch.Tensor:
    """partial statistics [rows, parts, 2] -> (mean, rstd) [rows, 2] of a `cols`-wide row (biased variance, nn.LayerNorm; rms: the
    T5 RMSNorm form (0, 1/sqrt(mean(x^2) + eps)))."""
    out = torch.empty((max(rows, 1), 2), dtype=torch.float32, device=partial.device)
    if rows:
        ctx.row_stats_finalize(partial[:rows], cols, eps, out, rms=rms)
    return out


def to_operand(ctx: _C.Context, x: torch.Tensor, p: Prec, *, pad_cols: Optional[int] = None) -> Opnd:
    """fp32 [rows, cols] -> Opnd (split kernel)."""
    assert x.dim() == 2
    if x.dtype != torch.float32:
        x = x.float()
    if x.stride(1) != 1:
        x = x.contiguous()
    rows, cols = x.shape
    o = Opnd(rows, cols if pad_cols is None else pad_cols, x.device, p.split)
    if rows:
        ctx.split(x, o.hi, o.lo, cols=cols, pad_cols=o.ld, dtype=p.dtype)
    return o


def norm(ctx: _C.Context, x: torch.Tensor, p: Prec, *, rows: int, cols: int, ldx: Optional[int] = None, w=None, b=None, eps=1e-5, rms=False,
         add=None, w2=None, b2=None, eps2=1e-5, want_f32=False, want2_f32=False, want16=False, out_f32=None, out_f8: bool = False,
         stats_eps: Optional[float] = None):
    """Returns (y1 fp32 | None, y2 fp32 | None, operands of the last norm | None[, (mean, rstd) [rows, 2] of y1 when stats_eps is given])."""
    dev = x.device
    ldx = cols if ldx is None else ldx
    o32 = out_f32 if out_f32 is not None else (torch.empty((rows, cols), dtype=torch.float32, device=dev) if want_f32 else None)
    o2 = torch.empty((rows, cols), dtype=torch.float32, device=dev) if want2_f32 else None
    o16 = Opnd(rows, cols, dev, p.split, f8=out_f8 and p.f8) if want16 else None
    st = torch.empty((max(rows, 1), 2), dtype=torch.float32, device=dev) if stats_eps is not None else None
    if rows:
        ctx.norm(x, rows=rows, cols=cols, ldx=ldx, w=w, b=b, eps=eps, rms=int(rms), add=add, w2=w2, b2=b2, eps2=eps2, out_f32=o32,
                 out2_f32=o2, out_hi=None if o16 is None else o16.hi, out_lo=None if o16 is None else o16.lo, dtype=p.dtype,
                 out_lo8=None if o16 is None else o16.lo8, out_hi8=None if o16 is None else o16.hi8, stats_out=st,
                 stats_eps=1e-5 if stats_eps is None else stats_eps)
    if stats_eps is not None:
        return o32, o2, o16, st
    return o32, o2, o16


def as_u8(mask: torch.Tensor) -> torch.Tensor:
    """bool -> uint8 view (same bytes; no copy) for the kernels' mask arguments."""
    if mask.dtype == torch.bool:
        return mask.contiguous().view(torch.uint8)
    return mask.to(torch.uint8).contiguous()
