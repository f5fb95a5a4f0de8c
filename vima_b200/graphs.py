"""CUDA-graph replay of a policy step (SURVEY.md section 7 step 9).

A policy step is ~230 kernel launches issued from Python through ctypes; at the 200M / 256-episode size the GPU never
starves, but at the small configurations (VIMA-20M, 64 episodes: ~2 ms of kernels) and in `forward_step` (33 rows per
episode) the launch path is the bound.  Shapes are static from step to step, every kernel takes its arguments by value
(tensor maps are `__grid_constant__` parameters, the tiny grouped GEMMs carry their descriptors in parameter space), and
nothing on the step synchronises with the host after the first call, so the whole step captures into one graph:

    g = GraphedStep(lambda obs: step(obs), example_obs)   # warms up, then captures on a side stream
    out = g(new_obs)                                        # copies new_obs into the static inputs, replays

The outputs are the tensors the captured call returned (static storage, overwritten by the next replay).

A graph holds the device pointers of the packed weights and parameters it read, so it is only valid for the weights and the
precision mode it was captured with.  Capture records them (`engine.record_weights`: every parameter of each module whose packed-
weight cache the step used) and keeps them alive; each replay first checks them and raises instead of launching when a parameter
was replaced or written in place, `refresh_weights` was called, or the precision mode changed.  Capture a new graph after a
weight update.
"""
from __future__ import annotations

from typing import Callable

import torch

from . import _C
from . import engine as eng
from .nn.action import _GroupedMLPs


def _map(fn, x, y=None):
    if isinstance(x, dict):
        return {k: _map(fn, v, None if y is None else y[k]) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return type(x)(_map(fn, v, None if y is None else y[i]) for i, v in enumerate(x))
    return fn(x) if y is None else fn(x, y)


def check_weights(weights: "eng.WeightState", precision: bool = True) -> None:
    """Raise before a replay that would read stale or freed weights (or run kernels of another precision mode)."""
    why = weights.changed()
    if why is None and precision and eng.prec().name != weights.precision:
        why = f"the precision mode changed from {weights.precision!r} to {eng.prec().name!r}"
    if why is not None:
        raise RuntimeError(f"{why} since this CUDA graph was captured; it would replay with the old ones. Capture it again.")


class GraphedStep:
    def __init__(self, fn: Callable, example_inputs, *, warmup: int = 3):
        """fn(inputs) -> nest of tensors; `example_inputs`: nest (dict / list / tensor) of CUDA tensors with the step's shapes."""
        self.fn = fn
        self.static_in = _map(lambda t: t.clone(), example_inputs)
        dev = next(iter(self._leaves(self.static_in))).device
        self.ctx = _C.Context.get(dev)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(max(warmup, 1)):  # packs weights, fills caches, runs the first-call host checks
                fn(self.static_in)
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        self.graph = torch.cuda.CUDAGraph()
        n0 = self.ctx.launches
        with eng.record_weights() as weights, torch.cuda.graph(self.graph):
            self.static_out = fn(self.static_in)
        self.weights = weights()
        self.kernels_per_replay = self.ctx.launches - n0  # vima:: kernels inside the graph (torch's own copies come on top)
        self.replays = 0

    @staticmethod
    def _leaves(x):
        if isinstance(x, dict):
            for v in x.values():
                yield from GraphedStep._leaves(v)
        elif isinstance(x, (list, tuple)):
            for v in x:
                yield from GraphedStep._leaves(v)
        else:
            yield x

    def __call__(self, inputs):
        check_weights(self.weights)
        if inputs is not self.static_in:
            _map(lambda dst, src: dst.copy_(src, non_blocking=True) if dst.data_ptr() != src.data_ptr() else dst, self.static_in, inputs)
        self.graph.replay()
        self.replays += 1
        return self.static_out

    def load_inputs(self, src):
        """Copy `src` (same nest; pinned host or device tensors) straight into the graph's static input buffers, asynchronously on
        the current stream; follow with `self(self.static_in)` to replay without a second device-to-device copy."""
        _map(lambda dst, s: dst.copy_(s, non_blocking=True), self.static_in, src)
        return self.static_in

    def describe(self) -> dict:
        return {"vima_kernels_per_replay": int(self.kernels_per_replay),
                "note": "the step is captured once (torch.cuda.CUDAGraph) and replayed; inputs are copied into static buffers"}


class GraphedSlotStep:
    """A policy's step_slots (or, with `act`, its act_slots) for one (S, Q), captured into a CUDA graph.  The slot state (len /
    n_valid / has_action / active) lives on the device and the step's kernels read it, so admissions and releases between replays
    take effect, and so do K/V pages taken between replays (the graph reads the device page table).  Warm-up runs the step (which
    advances the slots), so the state vectors, the fed-back action tokens, the page table, their host mirror, the page allocator
    and the sampler's draw counter are snapshotted first and restored afterwards; the K/V and mask columns warm-up wrote lie at or
    past each slot's `len` (in pages the slot owns, or skipped where it owns none) and are never read before a step overwrites them.

        g = policy.capture_step_slots(cache, obs, obs_mask, action)   # cache state unchanged
        out = g(obs, obs_mask, action)                                # = policy.step_slots(cache, obs, obs_mask, action)
        g = policy.capture_act_slots(cache, obs, obs_mask, sampler=s) # cache state and s unchanged
        actions, log_prob, entropy = g(obs, obs_mask)                 # = policy.act_slots(cache, obs, obs_mask, sampler=s)

    The step inputs are those of the policy's `_slot_step` after the cache: (obs_token, obs_mask, action_token) for VIMAPolicy,
    (obs_token, action_token) for the baselines, whose obs tokens are all valid; without the action token under `act`.  obs_token
    is (1,S,Q,E), or (1,S,E) with Q = 1.  The closed loop's action heads run on buffers the graph owns."""

    def __init__(self, policy, cache, obs_token: torch.Tensor, *inputs: torch.Tensor, warmup: int = 2, act: bool = False, sampler=None):
        self.policy, self.cache = policy, cache
        self.S, self.E = obs_token.shape[1], obs_token.shape[-1]
        self.Q = obs_token.shape[2] if obs_token.dim() == 4 else 1
        cache.check_step(self.S, self.Q, self.E, eng.prec())
        if act:
            self.static_in = [obs_token.clone()] + [t.clone() for t in inputs]
            # the graph's own head buffers: allocated by the warm-up outside the graph's pool, their addresses are baked into the
            # captured grouped GEMMs, so they must live as long as the graph
            self.grouped = _GroupedMLPs()
            step = lambda *a: policy._act_step(cache, *a, sampler=sampler, grouped=self.grouped)  # noqa: E731
        else:
            self.grouped = None
            self.static_in = [obs_token.clone()] + [t.clone() for t in inputs[:-1]] + [inputs[-1].float().clone()]
            step = lambda *a: policy._slot_step(cache, *a)  # noqa: E731
        dev = obs_token.device
        self.ctx = _C.Context.get(dev)
        saved = cache.state()
        saved_draws = None if sampler is None else sampler.counter.clone()
        try:
            side = torch.cuda.Stream(device=dev)
            side.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(side):
                for _ in range(max(warmup, 1)):  # packs weights, runs the first-call host checks, sets kernel attributes
                    step(*self.static_in)
            torch.cuda.current_stream(dev).wait_stream(side)
            torch.cuda.synchronize(dev)
            self.graph = torch.cuda.CUDAGraph()
            n0 = self.ctx.launches
            with eng.record_weights() as weights, torch.cuda.graph(self.graph):
                self.static_out = step(*self.static_in)
            self.weights = weights()
            self.kernels_per_replay = self.ctx.launches - n0
        finally:
            cache.restore(saved)
            if saved_draws is not None:
                sampler.counter.copy_(saved_draws)
            torch.cuda.synchronize(dev)
        self.replays = 0

    def __call__(self, obs_token: torch.Tensor, *inputs: torch.Tensor):
        if len(inputs) + 1 != len(self.static_in):
            raise ValueError(f"the graph was captured with {len(self.static_in)} step inputs, got {len(inputs) + 1}")
        check_weights(self.weights, precision=False)  # the cache refuses another precision mode (ValueError)
        self.cache.check_step(obs_token.shape[1], obs_token.shape[2] if obs_token.dim() == 4 else 1, obs_token.shape[-1], eng.prec())
        if tuple(obs_token.shape) != tuple(self.static_in[0].shape):
            raise ValueError(f"the graph was captured for obs_token {tuple(self.static_in[0].shape)}, got {tuple(obs_token.shape)}")
        self.cache.reserve_step(self.Q)  # the graph reads the device page table: pages taken here are the ones it writes and reads
        for dst, src in zip(self.static_in, (obs_token,) + inputs):
            if dst.data_ptr() != src.data_ptr():
                dst.copy_(src, non_blocking=True)
        self.graph.replay()
        self.replays += 1
        self.cache.advance_host(self.Q)
        return self.static_out
