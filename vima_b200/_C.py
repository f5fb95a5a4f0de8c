"""ctypes binding of libvima_b200.so (the C ABI in include/vima_b200.h).

There is NO fallback: if the library is missing or the device is not sm_90, every op raises.  torch is used
only to own device memory and streams; tensors cross the boundary as raw pointers.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_lib", "libvima_b200.so")

DT_F16, DT_BF16 = 0, 1
ACT_NONE, ACT_RELU, ACT_QUICKGELU, ACT_GELU, ACT_GELU_TANH = 0, 1, 2, 3, 4

c_void_p, c_int, c_float, c_i64 = C.c_void_p, C.c_int, C.c_float, C.c_int64


class GemmDesc(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32),
        ("M", c_int), ("N", c_int), ("K", c_int),
        ("a_hi", c_void_p), ("a_lo", c_void_p), ("lda", c_int),
        ("b_hi", c_void_p), ("b_lo", c_void_p), ("ldb", c_int),
        ("dtype", c_int), ("glu", c_int), ("act", c_int), ("acc_scale", c_float),
        ("bias", c_void_p),
        ("mul", c_void_p), ("ld_mul", c_int),
        ("residual", c_void_p), ("ld_res", c_int),
        ("out_f32", c_void_p), ("ld_o32", c_int),
        ("out_hi", c_void_p), ("out_lo", c_void_p), ("ld_o16", c_int),
        ("block_n", c_int),
        ("a_lo8", c_void_p), ("a_hi8", c_void_p), ("lda8", c_int),
        ("b_hi8", c_void_p), ("b_lo8", c_void_p), ("ldb8", c_int),
        ("out_lo8", c_void_p), ("out_hi8", c_void_p), ("ld_o8", c_int),
        # v5
        ("row_stats", c_void_p), ("ln_c1", c_void_p), ("ln_cols", c_int),
        ("res_stats", c_void_p), ("res_gamma", c_void_p), ("res_beta", c_void_p),
        ("stats_out", c_void_p), ("stats_parts", c_int),
    ]


class F32GemmGroup(C.Structure):
    _fields_ = [
        ("x", c_void_p), ("ldx", c_int),
        ("w", c_void_p), ("ldw", c_int),
        ("b", c_void_p),
        ("y", c_void_p), ("ldy", c_int),
        ("n", c_int), ("k", c_int),
    ]


class NormDesc(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32),
        ("x", c_void_p), ("rows", c_i64), ("cols", c_int), ("ldx", c_int),
        ("add", c_void_p), ("ld_add", c_int),
        ("w", c_void_p), ("b", c_void_p), ("eps", c_float), ("rms", c_int),
        ("w2", c_void_p), ("b2", c_void_p), ("eps2", c_float),
        ("out_f32", c_void_p), ("ld_o32", c_int),
        ("out2_f32", c_void_p), ("ld_o2", c_int),
        ("out_hi", c_void_p), ("out_lo", c_void_p), ("ld_o16", c_int),
        ("dtype", c_int),
        ("out_lo8", c_void_p), ("out_hi8", c_void_p), ("ld_o8", c_int),
        # v5
        ("stats_out", c_void_p), ("stats_eps", c_float),
    ]


class AttnDesc(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32),
        ("q_hi", c_void_p), ("q_lo", c_void_p), ("ldq", c_int),
        ("k_hi", c_void_p), ("k_lo", c_void_p), ("ldk", c_int),
        ("v_hi", c_void_p), ("v_lo", c_void_p), ("ldv", c_int),
        ("key_mask", c_void_p), ("rel_bias", c_void_p),
        ("o_hi", c_void_p), ("o_lo", c_void_p), ("ldo", c_int),
        ("B", c_int), ("H", c_int), ("Lq", c_int), ("Lk", c_int), ("D", c_int),
        ("scale", c_float), ("causal", c_int), ("dtype", c_int),
        ("o_lo8", c_void_p), ("o_hi8", c_void_p), ("ldo8", c_int),
        ("kv_batch_rows", c_int), ("mask_ld", c_int), ("q_pos0", c_int),
        # v5
        ("q_pos", c_void_p),
        # v6 tail (ABI version 5): paged k / v
        ("kv_pages", c_void_p), ("kv_page_ld", c_int), ("kv_pool_pages", c_int),
        # v7 tail (ABI version 5): per-batch key count
        ("kv_len", c_void_p),
    ]


KV_PAGE_TOKENS = 64  # include/vima_b200.h VIMA_KV_PAGE_TOKENS


class HeadSampleDesc(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32),
        ("logits", c_void_p), ("B", c_int), ("n_heads", c_int), ("head_off_dev", c_void_p),
        ("actions_in", c_void_p),
        ("greedy", c_int),
        ("seed", C.c_uint64), ("counter_dev", c_void_p),
        ("actions_out", c_void_p),
        ("log_prob", c_void_p), ("entropy", c_void_p), ("logits_norm", c_void_p),
    ]


_lib: Optional[C.CDLL] = None

EXPORTS = [
    "vima_abi_version", "vima_sizeof_gemm_desc", "vima_sizeof_norm_desc", "vima_sizeof_attn_desc", "vima_sizeof_f32_gemm_group", "vima_create", "vima_set_option", "vima_destroy", "vima_last_error", "vima_sm_count", "vima_launch_count",
    "vima_split_f32", "vima_pack_weight", "vima_gemm", "vima_glu_block_n", "vima_gemm_stats_parts", "vima_row_stats_finalize", "vima_gemm_f32_grouped", "vima_gemm_f32_grouped_host", "vima_norm",
    "vima_attention", "vima_small_attention", "vima_assemble_history", "vima_mask_cumsum", "vima_add_pos_embed",
    "vima_gather_prompt", "vima_patchify", "vima_vit_tokens", "vima_bbox_norm", "vima_fill_ee", "vima_max_u8",
    "vima_action_scale", "vima_action_postprocess", "vima_latent_attention", "vima_object_stats", "vima_crop_resize", "vima_head_select", "vima_gato_positions", "vima_pack_weight_f8", "vima_split_f8",
    "vima_slot_step_begin", "vima_slot_kv_append", "vima_slot_step_end", "vima_slot_kv_scatter", "vima_slot_admit_prefix",
    "vima_slot_kv_append_paged", "vima_slot_kv_scatter_paged", "vima_kv_copy_blocks", "vima_kv_pack_blocks",
    "vima_slot_assemble_history", "vima_slot_admit_history",
    "vima_head_sample", "vima_sizeof_head_sample_desc",
]


ABI_VERSION = 5  # include/vima_b200.h VIMA_B200_ABI_VERSION


def load_library() -> C.CDLL:
    """dlopen the in-tree library (works without a GPU: used by the CPU-side symbol test)."""
    global _lib
    if _lib is None:
        if not os.path.isfile(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: run `python -m vima_b200.build` (or __graft_entry__.build()). "
                "vima_b200 has no CPU / eager fallback."
            )
        _lib = C.CDLL(LIB_PATH)
        if _lib.vima_abi_version() != ABI_VERSION:  # descriptor structs below mirror include/vima_b200.h of this version
            got = _lib.vima_abi_version()
            _lib = None
            raise RuntimeError(f"{LIB_PATH} speaks C-ABI v{got}, this package needs v{ABI_VERSION}: rebuild with `python -m vima_b200.build`")
        for name, mirror in (("gemm_desc", GemmDesc), ("norm_desc", NormDesc), ("attn_desc", AttnDesc), ("f32_gemm_group", F32GemmGroup),
                             ("head_sample_desc", HeadSampleDesc)):
            want = getattr(_lib, f"vima_sizeof_{name}")()
            if want != C.sizeof(mirror):  # the ctypes mirrors above and include/vima_b200.h have drifted apart
                _lib = None
                raise RuntimeError(f"ctypes mirror of vima_{name} is {C.sizeof(mirror)} bytes, the library's struct is {want}")
        _lib.vima_last_error.restype = C.c_char_p
        _lib.vima_launch_count.restype = c_i64
        _lib.vima_create.argtypes = [C.POINTER(c_void_p), c_int]
        _lib.vima_destroy.argtypes = [c_void_p]
        _lib.vima_last_error.argtypes = [c_void_p]
        _lib.vima_launch_count.argtypes = [c_void_p]
        _lib.vima_sm_count.argtypes = [c_void_p]
        _lib.vima_set_option.argtypes = [c_void_p, C.c_char_p, C.c_char_p]
    return _lib


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()




class Context:
    """One per device.  Every method enqueues kernels on torch's current stream of THAT device."""

    _by_device: dict = {}

    def __init__(self, device: int):
        self.lib = load_library()
        h = c_void_p()
        rc = self.lib.vima_create(C.byref(h), int(device))
        if rc != 0:
            raise RuntimeError(
                f"vima_create(device={device}) failed with code {rc}: vima_b200 needs an sm_90 (H100) device; "
                "there is no CPU or non-Hopper fallback"
            )
        self.h = h
        self.device = int(device)
        self.sm_count = self.lib.vima_sm_count(h)

    @classmethod
    def get(cls, device) -> "Context":
        if isinstance(device, torch.device):
            if device.type != "cuda":
                raise RuntimeError(f"vima_b200 runs on CUDA devices only (got {device}); there is no CPU path")
            device = device.index if device.index is not None else torch.cuda.current_device()
        if device not in cls._by_device:
            cls._by_device[device] = Context(device)
        return cls._by_device[device]

    def _s(self) -> int:
        """torch's current stream ON THIS CONTEXT'S DEVICE (not on the thread's current device)."""
        return torch.cuda.current_stream(self.device).cuda_stream

    def _ck(self, rc: int, what: str):
        if rc != 0:
            msg = self.lib.vima_last_error(self.h)
            raise RuntimeError(f"{what} failed (code {rc}): {msg.decode() if msg else ''}")

    def set_option(self, key: str, value: str) -> None:
        """Kernel selection of this context: attn = tc | mma, attn_tail = kernel | off, epi_prefetch = 1 | 0, attn_bias = auto | tc
        (relative-bias attention, i.e. the T5 encoder, on the K/V-streaming wgmma kernel only past the resident-K/V kernel's
        shared memory, or at every length), gemm_wide = 1 | 0 (f16f8 GEMMs with 128-wide tiles and N % 256 == 0 on 128 x 256
        tiles, or on the 128-wide kernel)."""
        self._ck(self.lib.vima_set_option(self.h, key.encode(), str(value).encode()), "set_option")

    @property
    def launches(self) -> int:
        return int(self.lib.vima_launch_count(self.h))

    # ---------------------------------------------------------------- operand prep
    def split(self, x: torch.Tensor, hi: torch.Tensor, lo: Optional[torch.Tensor], *, cols=None, pad_cols=None, scale=1.0, dtype=DT_F16):
        """x fp32 [rows, >=cols] -> hi/lo 16-bit [rows, ld16]."""
        assert x.dtype == torch.float32 and x.dim() == 2 and x.stride(1) == 1
        cols = x.shape[1] if cols is None else cols
        pad_cols = cols if pad_cols is None else pad_cols
        self._ck(self.lib.vima_split_f32(self.h, c_void_p(x.data_ptr()), c_i64(x.shape[0]), cols, x.stride(0), c_void_p(hi.data_ptr()),
                                         c_void_p(_ptr(lo)), hi.stride(0), pad_cols, c_float(scale), dtype, c_void_p(self._s())), "split_f32")

    def pack_weight(self, w: torch.Tensor, hi: torch.Tensor, lo: Optional[torch.Tensor], *, transposed: bool, scale=1.0, dtype=DT_F16):
        assert w.dtype == torch.float32 and w.dim() == 2 and w.stride(1) == 1
        n, k = (w.shape[1], w.shape[0]) if transposed else (w.shape[0], w.shape[1])
        assert hi.shape[0] >= n
        self._ck(self.lib.vima_pack_weight(self.h, c_void_p(w.data_ptr()), n, k, int(transposed), w.stride(0), c_void_p(hi.data_ptr()),
                                           c_void_p(_ptr(lo)), hi.stride(0), c_float(scale), dtype, c_void_p(self._s())), "pack_weight")

    def pack_weight_f8(self, w: torch.Tensor, hi8: torch.Tensor, lo8: torch.Tensor, *, transposed: bool, scale=1.0):
        n, k = (w.shape[1], w.shape[0]) if transposed else (w.shape[0], w.shape[1])
        self._ck(self.lib.vima_pack_weight_f8(self.h, c_void_p(w.data_ptr()), n, k, int(transposed), w.stride(0), c_void_p(hi8.data_ptr()),
                                              c_void_p(lo8.data_ptr()), hi8.stride(0), c_float(scale), c_void_p(self._s())), "pack_weight_f8")

    def split_f8(self, x: torch.Tensor, lo8: torch.Tensor, hi8: torch.Tensor):
        self._ck(self.lib.vima_split_f8(self.h, c_void_p(x.data_ptr()), c_i64(x.shape[0]), x.shape[1], x.stride(0), c_void_p(lo8.data_ptr()),
                                        c_void_p(hi8.data_ptr()), lo8.stride(0), c_void_p(self._s())), "split_f8")

    def gemm_stats_parts(self, N: int, glu: int, block_n: int = 0) -> int:
        return int(self.lib.vima_gemm_stats_parts(int(N), int(glu), int(block_n)))

    def row_stats_finalize(self, partial: torch.Tensor, cols: int, eps: float, stats: torch.Tensor, rms: bool = False):
        """partial fp32 [rows, parts, 2] -> stats fp32 [rows, 2] = (mean, rstd)  (rms: (0, 1/sqrt(mean(x^2) + eps)))."""
        rows, parts, _ = partial.shape
        self._ck(self.lib.vima_row_stats_finalize(self.h, c_void_p(partial.data_ptr()), c_i64(rows), int(parts), int(cols), c_float(eps),
                                                  int(rms), c_void_p(stats.data_ptr()), c_void_p(self._s())), "row_stats_finalize")

    def glu_block_n(self, n_out: int) -> int:
        return int(self.lib.vima_glu_block_n(int(n_out)))

    # ---------------------------------------------------------------- GEMMs
    def gemm(self, *, M, N, K, a_hi, a_lo, lda, b_hi, b_lo, ldb, dtype=DT_F16, glu=0, act=ACT_NONE, acc_scale=1.0, bias=None,
             mul=None, residual=None, out_f32=None, out_hi=None, out_lo=None, ld_o16=0, block_n=0, a_lo8=None, a_hi8=None, b_hi8=None,
             b_lo8=None, out_lo8=None, out_hi8=None, row_stats=None, ln_c1=None, ln_cols=0, res_stats=None, res_gamma=None, res_beta=None,
             stats_out=None):
        d = GemmDesc()
        d.struct_size = C.sizeof(GemmDesc)
        d.M, d.N, d.K = int(M), int(N), int(K)
        d.a_hi, d.a_lo, d.lda = a_hi.data_ptr(), _ptr(a_lo), int(lda)
        d.b_hi, d.b_lo, d.ldb = b_hi.data_ptr(), _ptr(b_lo), int(ldb)
        d.dtype, d.glu, d.act, d.acc_scale = dtype, int(glu), int(act), float(acc_scale)
        d.bias = _ptr(bias)
        d.mul, d.ld_mul = _ptr(mul), (mul.stride(0) if mul is not None else 0)
        d.residual, d.ld_res = _ptr(residual), (residual.stride(0) if residual is not None else 0)
        d.out_f32, d.ld_o32 = _ptr(out_f32), (out_f32.stride(0) if out_f32 is not None else 0)
        d.out_hi, d.out_lo, d.ld_o16 = _ptr(out_hi), _ptr(out_lo), int(ld_o16 or (out_hi.stride(0) if out_hi is not None else 0))
        d.block_n = int(block_n)
        d.a_lo8, d.a_hi8, d.lda8 = _ptr(a_lo8), _ptr(a_hi8), (a_lo8.stride(0) if a_lo8 is not None else 0)
        d.b_hi8, d.b_lo8, d.ldb8 = _ptr(b_hi8), _ptr(b_lo8), (b_hi8.stride(0) if b_hi8 is not None else 0)
        d.out_lo8, d.out_hi8, d.ld_o8 = _ptr(out_lo8), _ptr(out_hi8), (out_lo8.stride(0) if out_lo8 is not None else 0)
        d.row_stats, d.ln_c1, d.ln_cols = _ptr(row_stats), _ptr(ln_c1), int(ln_cols)
        d.res_stats, d.res_gamma, d.res_beta = _ptr(res_stats), _ptr(res_gamma), _ptr(res_beta)
        d.stats_out, d.stats_parts = _ptr(stats_out), (stats_out.shape[1] if stats_out is not None else 0)
        self._ck(self.lib.vima_gemm(self.h, C.byref(d), c_void_p(self._s())), "gemm")

    def gemm_f32_grouped(self, groups_dev: torch.Tensor, n_groups: int, M: int, max_n: int, act: int):
        self._ck(self.lib.vima_gemm_f32_grouped(self.h, c_void_p(groups_dev.data_ptr()), n_groups, M, max_n, act, c_void_p(self._s())),
                 "gemm_f32_grouped")

    def gemm_f32_grouped_host(self, groups_arr, n_groups: int, M: int, max_n: int, act: int):
        """groups_arr: ctypes array of F32GemmGroup in host memory (travels by value: CUDA-graph safe)."""
        self._ck(self.lib.vima_gemm_f32_grouped_host(self.h, groups_arr, n_groups, M, max_n, act, c_void_p(self._s())), "gemm_f32_grouped_host")

    # ---------------------------------------------------------------- norm / attention
    def norm(self, x, *, rows, cols, ldx, w=None, b=None, eps=1e-5, rms=0, add=None, w2=None, b2=None, eps2=1e-5, out_f32=None,
             out2_f32=None, out_hi=None, out_lo=None, dtype=DT_F16, out_lo8=None, out_hi8=None, stats_out=None, stats_eps=1e-5):
        d = NormDesc()
        d.struct_size = C.sizeof(NormDesc)
        d.x, d.rows, d.cols, d.ldx = x.data_ptr(), int(rows), int(cols), int(ldx)
        d.add, d.ld_add = _ptr(add), (add.stride(0) if add is not None else 0)
        d.w, d.b, d.eps, d.rms = _ptr(w), _ptr(b), float(eps), int(rms)
        d.w2, d.b2, d.eps2 = _ptr(w2), _ptr(b2), float(eps2)
        d.out_f32, d.ld_o32 = _ptr(out_f32), (out_f32.stride(0) if out_f32 is not None else 0)
        d.out2_f32, d.ld_o2 = _ptr(out2_f32), (out2_f32.stride(0) if out2_f32 is not None else 0)
        d.out_hi, d.out_lo, d.ld_o16 = _ptr(out_hi), _ptr(out_lo), (out_hi.stride(0) if out_hi is not None else 0)
        d.dtype = dtype
        d.out_lo8, d.out_hi8, d.ld_o8 = _ptr(out_lo8), _ptr(out_hi8), (out_lo8.stride(0) if out_lo8 is not None else 0)
        d.stats_out, d.stats_eps = _ptr(stats_out), float(stats_eps)
        self._ck(self.lib.vima_norm(self.h, C.byref(d), c_void_p(self._s())), "norm")

    def attention(self, *, q, k, v, o, B, H, Lq, Lk, D, scale, causal=False, key_mask=None, rel_bias=None, dtype=DT_F16, o8=None,
                  kv_batch_rows=0, mask_ld=0, q_pos0=0, q_pos=None, kv_pages=None, kv_pool_pages=0, kv_len=None):
        """q, k, v, o: (hi, lo|None, ld, column offset) tuples over 16-bit operand buffers.  q_pos: int32 [B] on the device, the
        causal position of each batch element's first query row (its key count is then q_pos[b] + Lq; Lk is the capacity).
        kv_pages: int32 [B, page_ld] on the device, paged k / v: key j of element b is row kv_pages[b, j // 64] * 64 + j % 64 of k / v,
        a pool of kv_pool_pages pages.  kv_len: int32 [B] on the device (non-causal, no q_pos): element b attends keys
        [0, clamp(kv_len[b], 1, Lk))."""
        es = 2

        def at(t, off):
            return None if t is None else t.data_ptr() + off * es

        d = AttnDesc()
        d.struct_size = C.sizeof(AttnDesc)
        d.q_hi, d.q_lo, d.ldq = at(q[0], q[3]), at(q[1], q[3]), q[2]
        d.k_hi, d.k_lo, d.ldk = at(k[0], k[3]), at(k[1], k[3]), k[2]
        d.v_hi, d.v_lo, d.ldv = at(v[0], v[3]), at(v[1], v[3]), v[2]
        d.o_hi, d.o_lo, d.ldo = at(o[0], o[3]), at(o[1], o[3]), o[2]
        d.key_mask, d.rel_bias = _ptr(key_mask), _ptr(rel_bias)
        d.B, d.H, d.Lq, d.Lk, d.D = int(B), int(H), int(Lq), int(Lk), int(D)
        d.scale, d.causal, d.dtype = float(scale), int(causal), dtype
        d.kv_batch_rows, d.mask_ld, d.q_pos0 = int(kv_batch_rows), int(mask_ld), int(q_pos0)
        if q_pos is not None:
            assert q_pos.dtype == torch.int32 and q_pos.is_contiguous() and q_pos.numel() >= B
            d.q_pos = q_pos.data_ptr()
        if kv_pages is not None:
            assert kv_pages.dtype == torch.int32 and kv_pages.dim() == 2 and kv_pages.is_contiguous() and kv_pages.shape[0] >= B
            d.kv_pages, d.kv_page_ld, d.kv_pool_pages = kv_pages.data_ptr(), kv_pages.shape[1], int(kv_pool_pages)
        if kv_len is not None:
            assert kv_len.dtype == torch.int32 and kv_len.is_contiguous() and kv_len.numel() >= B
            d.kv_len = kv_len.data_ptr()
        if o8 is not None:  # (lo8, hi8) uint8 [rows, ld8]
            d.o_lo8, d.o_hi8, d.ldo8 = o8[0].data_ptr(), o8[1].data_ptr(), o8[0].stride(0)
        self._ck(self.lib.vima_attention(self.h, C.byref(d), c_void_p(self._s())), "attention")

    def small_attention(self, qkv, *, N, S, H, W, scale, o_hi, o_lo, o_f32=None, dtype=DT_F16):
        self._ck(self.lib.vima_small_attention(self.h, c_void_p(qkv.data_ptr()), qkv.stride(0), c_i64(N), S, H, W, c_float(scale),
                                               c_void_p(_ptr(o_hi)), c_void_p(_ptr(o_lo)), (o_hi.stride(0) if o_hi is not None else W),
                                               c_void_p(_ptr(o_f32)), dtype, c_void_p(self._s())), "small_attention")

    # ---------------------------------------------------------------- token assembly
    def assemble_history(self, obs, obs_mask_u8, action, tokens, masks_bl, pos_bl):
        T, B, Q, E = obs.shape
        La = 0 if action is None else action.shape[0]
        self._ck(self.lib.vima_assemble_history(self.h, c_void_p(obs.data_ptr()), c_void_p(obs_mask_u8.data_ptr()), c_void_p(_ptr(action)), T, B,
                                                Q, E, La, c_void_p(tokens.data_ptr()), c_void_p(masks_bl.data_ptr()),
                                                c_void_p(pos_bl.data_ptr()), c_void_p(self._s())), "assemble_history")

    def mask_cumsum(self, mask_u8, pos):
        B, L = mask_u8.shape
        self._ck(self.lib.vima_mask_cumsum(self.h, c_void_p(mask_u8.data_ptr()), B, L, c_void_p(pos.data_ptr()), c_void_p(self._s())), "mask_cumsum")

    # ---------------------------------------------------------------- slot decode (per-slot int32 state vectors on the device)
    def slot_step_begin(self, obs, obs_mask_u8, action, *, Lmax, len_, n_valid, has_action, active, tokens, step_mask, pos, q_pos, slot_mask):
        """obs fp32 [S, Q, E], obs_mask uint8 [S, Q], action fp32 [S, E] -> tokens [S*(Q+1), E], step_mask [S, Q+1], pos int64 [S, Q+1],
        q_pos int32 [S]; writes the step's columns of slot_mask [S, Lmax]."""
        S, Q, E = obs.shape
        self._ck(self.lib.vima_slot_step_begin(self.h, c_void_p(obs.data_ptr()), c_void_p(obs_mask_u8.data_ptr()), c_void_p(action.data_ptr()),
                                               S, Q, E, int(Lmax), c_void_p(len_.data_ptr()), c_void_p(n_valid.data_ptr()),
                                               c_void_p(has_action.data_ptr()), c_void_p(active.data_ptr()), c_void_p(tokens.data_ptr()),
                                               c_void_p(step_mask.data_ptr()), c_void_p(pos.data_ptr()), c_void_p(q_pos.data_ptr()),
                                               c_void_p(slot_mask.data_ptr()), c_void_p(self._s())), "slot_step_begin")

    def slot_kv_append(self, qkv_hi, qkv_lo, ld_qkv, col0, width, S, Lq, q_pos, kv_hi, kv_lo, ld_kv, Lmax):
        self._ck(self.lib.vima_slot_kv_append(self.h, c_void_p(qkv_hi.data_ptr()), c_void_p(_ptr(qkv_lo)), int(ld_qkv), int(col0), int(width),
                                              int(S), int(Lq), c_void_p(q_pos.data_ptr()), c_void_p(kv_hi.data_ptr()), c_void_p(_ptr(kv_lo)),
                                              int(ld_kv), int(Lmax), c_void_p(self._s())), "slot_kv_append")

    def slot_kv_append_paged(self, qkv_hi, qkv_lo, ld_qkv, col0, width, S, Lq, q_pos, kv_hi, kv_lo, ld_kv, pages, pool_pages):
        """slot_kv_append into a paged cache: pages int32 [S, page_ld] (device) of page indices into kv [pool_pages*64, ld_kv]."""
        assert pages.dtype == torch.int32 and pages.dim() == 2 and pages.is_contiguous()
        self._ck(self.lib.vima_slot_kv_append_paged(self.h, c_void_p(qkv_hi.data_ptr()), c_void_p(_ptr(qkv_lo)), int(ld_qkv), int(col0),
                                                    int(width), int(S), int(Lq), c_void_p(q_pos.data_ptr()), c_void_p(kv_hi.data_ptr()),
                                                    c_void_p(_ptr(kv_lo)), int(ld_kv), c_void_p(pages.data_ptr()), pages.shape[1],
                                                    int(pool_pages), c_void_p(self._s())), "slot_kv_append_paged")

    def slot_step_end(self, x, S, Q, E, step_mask, *, len_, n_valid, has_action, active, out):
        """x fp32 [S*(Q+1), >=E] -> out [S, E] (each slot's prediction row); advances the active slots' state."""
        self._ck(self.lib.vima_slot_step_end(self.h, c_void_p(x.data_ptr()), x.stride(0), int(S), int(Q), int(E), c_void_p(step_mask.data_ptr()),
                                             c_void_p(len_.data_ptr()), c_void_p(n_valid.data_ptr()), c_void_p(has_action.data_ptr()),
                                             c_void_p(active.data_ptr()), c_void_p(out.data_ptr()), c_void_p(self._s())), "slot_step_end")

    def slot_kv_scatter(self, qkv_hi, qkv_lo, ld_qkv, col0, width, n, Lq, slots, kv_hi, kv_lo, ld_kv, Lmax):
        """Prefill rows (j, r) of qkv [n*Lq, ld_qkv], columns [col0, col0+width) -> rows slots[j]*Lmax + r of kv; slots int32 [n]."""
        assert slots.dtype == torch.int32 and slots.is_contiguous() and slots.numel() >= n
        self._ck(self.lib.vima_slot_kv_scatter(self.h, c_void_p(qkv_hi.data_ptr()), c_void_p(_ptr(qkv_lo)), int(ld_qkv), int(col0), int(width),
                                               int(n), int(Lq), c_void_p(slots.data_ptr()), c_void_p(kv_hi.data_ptr()), c_void_p(_ptr(kv_lo)),
                                               int(ld_kv), int(Lmax), c_void_p(self._s())), "slot_kv_scatter")

    def slot_kv_scatter_paged(self, qkv_hi, qkv_lo, ld_qkv, col0, width, n, Lq, slots, kv_hi, kv_lo, ld_kv, pages, pool_pages):
        """slot_kv_scatter into a paged cache: prefill row (j, r) -> row pages[slots[j], r // 64] * 64 + r % 64 of kv."""
        assert slots.dtype == torch.int32 and slots.is_contiguous() and slots.numel() >= n
        assert pages.dtype == torch.int32 and pages.dim() == 2 and pages.is_contiguous()
        self._ck(self.lib.vima_slot_kv_scatter_paged(self.h, c_void_p(qkv_hi.data_ptr()), c_void_p(_ptr(qkv_lo)), int(ld_qkv), int(col0),
                                                     int(width), int(n), int(Lq), c_void_p(slots.data_ptr()), c_void_p(kv_hi.data_ptr()),
                                                     c_void_p(_ptr(kv_lo)), int(ld_kv), c_void_p(pages.data_ptr()), pages.shape[1],
                                                     int(pool_pages), c_void_p(self._s())), "slot_kv_scatter_paged")

    def slot_admit_prefix(self, slots, prompt_mask_u8, Lmax, slot_mask, *, len_, n_valid, has_action, active):
        """slots int32 [n], prompt_mask uint8 [n, Lp] -> mask columns [0, Lp] of the admitted slots and their fresh state."""
        n, Lp = prompt_mask_u8.shape
        assert slots.dtype == torch.int32 and slots.numel() == n and prompt_mask_u8.is_contiguous()
        self._ck(self.lib.vima_slot_admit_prefix(self.h, c_void_p(slots.data_ptr()), int(n), c_void_p(prompt_mask_u8.data_ptr()), int(Lp), int(Lmax),
                                                 c_void_p(slot_mask.data_ptr()), c_void_p(len_.data_ptr()), c_void_p(n_valid.data_ptr()),
                                                 c_void_p(has_action.data_ptr()), c_void_p(active.data_ptr()), c_void_p(self._s())),
                 "slot_admit_prefix")

    def slot_assemble_history(self, obs, obs_mask_u8, action, steps, P, tokens, mask, pos):
        """obs fp32 (T, n, Q, E), obs_mask uint8 (T, n, Q) | None (every obs token valid), action fp32 (T, n, E), steps int32 [n]
        (device) -> rows [P, L) of tokens (L, n, E) and columns [P, L) of mask uint8 / pos int64 [n, L], each episode's own history
        (columns [0, P) of mask are read for the position base)."""
        T, n, Q, E = obs.shape
        L = tokens.shape[0]
        assert steps.dtype == torch.int32 and steps.numel() == n and action.shape == (T, n, E) and tokens.shape == (L, n, E)
        assert mask.shape == (n, L) and pos.shape == (n, L) and all(t.is_contiguous() for t in (obs, action, tokens, mask, pos, steps))
        assert obs_mask_u8 is None or (obs_mask_u8.shape == (T, n, Q) and obs_mask_u8.is_contiguous())
        if L == P or n == 0:  # no history column to write
            return
        self._ck(self.lib.vima_slot_assemble_history(self.h, c_void_p(_ptr(obs) if T else None), c_void_p(_ptr(obs_mask_u8) if T else None),
                                                     c_void_p(_ptr(action) if T else None), c_void_p(steps.data_ptr()), int(T), int(n), int(Q),
                                                     int(E), int(P), int(L), c_void_p(tokens.data_ptr()), c_void_p(mask.data_ptr()),
                                                     c_void_p(pos.data_ptr()), c_void_p(self._s())), "slot_assemble_history")

    def slot_admit_history(self, slots, steps, Q, P, mask, action, Lmax, slot_mask, *, len_, n_valid, has_action, active, action_token):
        """slots / steps int32 [n] (device), mask uint8 [n, L] (assembled), action fp32 (T, n, E) -> the admitted slots' mask rows of
        slot_mask [S, Lmax], their state (len, n_valid, has_action, active) and fed-back action rows of action_token [S, E]."""
        n, L = mask.shape
        T, E = action.shape[0], action.shape[2]
        S = slot_mask.shape[0]
        assert slots.dtype == torch.int32 and steps.dtype == torch.int32 and slots.numel() == n and steps.numel() == n
        assert mask.is_contiguous() and action.is_contiguous() and action.shape[1] == n and action_token.shape == (S, E)
        self._ck(self.lib.vima_slot_admit_history(self.h, c_void_p(slots.data_ptr()), c_void_p(steps.data_ptr()), int(n), int(S), int(T), int(Q),
                                                  int(P), int(L), c_void_p(_ptr(mask) if L else None), c_void_p(_ptr(action) if T else None),
                                                  int(E), int(Lmax), c_void_p(slot_mask.data_ptr()), c_void_p(len_.data_ptr()),
                                                  c_void_p(n_valid.data_ptr()), c_void_p(has_action.data_ptr()), c_void_p(active.data_ptr()),
                                                  c_void_p(action_token.data_ptr()), c_void_p(self._s())), "slot_admit_history")

    def kv_copy_blocks(self, bufs, row_bytes, src_row0, dst_row0, block_rows, buf_rows):
        """Block i of block_rows rows at row src_row0[i] -> row dst_row0[i] in every buffer whose base address bufs (int64 [n_buf],
        device) lists; src_row0 / dst_row0 int64 [n_blocks] (device).  Blocks starting outside [0, buf_rows - block_rows] are skipped."""
        assert bufs.dtype == torch.int64 and src_row0.dtype == torch.int64 and dst_row0.dtype == torch.int64
        assert src_row0.is_contiguous() and dst_row0.is_contiguous() and src_row0.numel() == dst_row0.numel()
        self._ck(self.lib.vima_kv_copy_blocks(self.h, c_void_p(bufs.data_ptr()), int(bufs.numel()), c_i64(row_bytes),
                                              c_void_p(src_row0.data_ptr()), c_void_p(dst_row0.data_ptr()), int(src_row0.numel()),
                                              int(block_rows), c_i64(buf_rows), c_void_p(self._s())), "kv_copy_blocks")

    def kv_pack_blocks(self, bufs, row_bytes, row0, block_rows, buf_rows, packed, unpack):
        """Block i of block_rows rows at row row0[i] of every buffer whose base address bufs (int64 [n_buf], device) lists <-> packed
        [block][buffer][block_rows][row_bytes] (a device tensor); unpack=False packs, True unpacks.  row0 int64 [n_blocks] (device).
        Blocks starting outside [0, buf_rows - block_rows] are skipped."""
        assert bufs.dtype == torch.int64 and row0.dtype == torch.int64 and row0.is_contiguous() and packed.is_contiguous()
        assert packed.numel() * packed.element_size() >= row0.numel() * bufs.numel() * block_rows * row_bytes
        self._ck(self.lib.vima_kv_pack_blocks(self.h, c_void_p(bufs.data_ptr()), int(bufs.numel()), c_i64(row_bytes), c_void_p(row0.data_ptr()),
                                              int(row0.numel()), int(block_rows), c_i64(buf_rows), c_void_p(packed.data_ptr()), int(bool(unpack)),
                                              c_void_p(self._s())), "kv_pack_blocks")

    def add_pos_embed(self, tok, stride_b, stride_l, ids, table, B, L, E, *, out_f32=None, hi=None, lo=None, dtype=DT_F16, err_flag=None):
        self._ck(self.lib.vima_add_pos_embed(self.h, c_void_p(tok.data_ptr()), c_i64(stride_b), c_i64(stride_l), c_void_p(ids.data_ptr()),
                                             c_void_p(table.data_ptr()), table.shape[0], B, L, E, c_void_p(_ptr(out_f32)), c_void_p(_ptr(hi)),
                                             c_void_p(_ptr(lo)), (hi.stride(0) if hi is not None else 0), dtype, c_void_p(_ptr(err_flag)),
                                             c_void_p(self._s())), "add_pos_embed")

    def gather_prompt(self, kind, index, word_ids, word_table, img_emb, img_mask_u8, B, Lp, D, out, mask_out):
        self._ck(self.lib.vima_gather_prompt(self.h, c_void_p(kind.data_ptr()), c_void_p(index.data_ptr()), c_void_p(word_ids.data_ptr()),
                                             c_void_p(word_table.data_ptr()), c_void_p(img_emb.data_ptr()), c_void_p(img_mask_u8.data_ptr()),
                                             B, Lp, D, c_void_p(out.data_ptr()), c_void_p(mask_out.data_ptr()), c_void_p(self._s())),
                 "gather_prompt")

    # ---------------------------------------------------------------- object encoder front end
    def patchify(self, img_u8, N, H, W, P, hi, lo, dtype=DT_F16):
        self._ck(self.lib.vima_patchify(self.h, c_void_p(img_u8.data_ptr()), c_i64(N), H, W, P, c_void_p(hi.data_ptr()), c_void_p(_ptr(lo)),
                                        hi.stride(0), dtype, c_void_p(self._s())), "patchify")

    def gato_positions(self, prompt_mask_u8, L, mask_out, pos_out):
        B, Lp = prompt_mask_u8.shape
        self._ck(self.lib.vima_gato_positions(self.h, c_void_p(prompt_mask_u8.data_ptr()), B, Lp, L, c_void_p(mask_out.data_ptr()),
                                              c_void_p(pos_out.data_ptr()), c_void_p(self._s())), "gato_positions")

    def vit_tokens(self, patch_out, cls, pos, N, S, W, out):
        self._ck(self.lib.vima_vit_tokens(self.h, c_void_p(patch_out.data_ptr()), c_void_p(_ptr(cls)), c_void_p(pos.data_ptr()), c_i64(N),
                                          S, W, c_void_p(out.data_ptr()), c_void_p(self._s())), "vit_tokens")

    def bbox_norm(self, bbox_i64, n, out):
        self._ck(self.lib.vima_bbox_norm(self.h, c_void_p(bbox_i64.data_ptr()), c_i64(n), c_void_p(out.data_ptr()), c_void_p(self._s())), "bbox_norm")

    def fill_ee(self, ee_i64, table, n_te, Q, hi, lo, col0, n_pad, dtype=DT_F16):
        self._ck(self.lib.vima_fill_ee(self.h, c_void_p(ee_i64.data_ptr()), c_void_p(table.data_ptr()), c_i64(n_te), Q, c_void_p(hi.data_ptr()),
                                       c_void_p(_ptr(lo)), hi.stride(0), col0, n_pad, dtype, c_void_p(self._s())), "fill_ee")

    def max_u8(self, x_u8, out_max_i32):
        self._ck(self.lib.vima_max_u8(self.h, c_void_p(x_u8.data_ptr()), c_i64(x_u8.numel()), c_void_p(out_max_i32.data_ptr()),
                                      c_void_p(self._s())), "max_u8")

    # ---------------------------------------------------------------- action heads
    def action_scale(self, idx_i64, n, width, bins, out):
        self._ck(self.lib.vima_action_scale(self.h, c_void_p(idx_i64.data_ptr()), c_i64(n), width, c_void_p(bins.data_ptr()),
                                            c_void_p(out.data_ptr()), c_void_p(self._s())), "action_scale")

    def object_stats(self, segm, n_img, H, W, ids_i64, n_obj, ids_per_image, stats_i32):
        self._ck(self.lib.vima_object_stats(self.h, c_void_p(segm.data_ptr()), segm.element_size(), n_img, H, W, c_void_p(ids_i64.data_ptr()),
                                            n_obj, int(ids_per_image), c_void_p(stats_i32.data_ptr()), c_void_p(self._s())), "object_stats")

    def crop_resize(self, rgb_u8, n_img, H, W, stats_i32, n_obj, crops, bbox, mask, n_valid=None):
        self._ck(self.lib.vima_crop_resize(self.h, c_void_p(rgb_u8.data_ptr()), n_img, H, W, c_void_p(stats_i32.data_ptr()), n_obj,
                                           c_void_p(crops.data_ptr()), c_void_p(bbox.data_ptr()), c_void_p(mask.data_ptr()),
                                           c_void_p(_ptr(n_valid)), c_void_p(self._s())), "crop_resize")

    def latent_attention(self, *, q, ldq, q_batch_stride, k, ldk, v, ldv, o, ldo, N, Lq, Lk, H, d, scale):
        self._ck(self.lib.vima_latent_attention(self.h, c_void_p(q.data_ptr()), ldq, c_i64(q_batch_stride), c_void_p(k.data_ptr()), ldk,
                                                c_void_p(v.data_ptr()), ldv, c_void_p(o.data_ptr()), ldo, c_i64(N), Lq, Lk, H, d,
                                                C.c_float(scale), c_void_p(self._s())), "latent_attention")

    def action_postprocess(self, idx_i64, n, width, bins, lo, hi, bound_stride, out):
        self._ck(self.lib.vima_action_postprocess(self.h, c_void_p(idx_i64.data_ptr()), c_i64(n), width, c_void_p(bins.data_ptr()),
                                                  c_void_p(lo.data_ptr()), c_void_p(hi.data_ptr()), bound_stride, c_void_p(out.data_ptr()),
                                                  c_void_p(self._s())), "action_postprocess")

    def head_select(self, logits, B, n_heads, head_off_i32, logits_norm, modes):
        self._ck(self.lib.vima_head_select(self.h, c_void_p(logits.data_ptr()), B, n_heads, c_void_p(head_off_i32.data_ptr()),
                                           c_void_p(_ptr(logits_norm)), c_void_p(modes.data_ptr()), c_void_p(self._s())), "head_select")

    def head_sample(self, logits, B, n_heads, head_off_i32, *, actions_in=None, greedy=False, seed=0, counter=None, actions_out=None,
                    log_prob=None, entropy=None, logits_norm=None):
        """vima_head_sample: score actions_in (int64 [B, n_heads]), or choose the mode (greedy) or a Philox draw at the device draw
        index `counter` (one uint64, advanced by the call) into actions_out."""
        d = HeadSampleDesc()
        d.struct_size = C.sizeof(HeadSampleDesc)
        d.logits, d.B, d.n_heads, d.head_off_dev = logits.data_ptr(), int(B), int(n_heads), head_off_i32.data_ptr()
        d.actions_in, d.greedy = _ptr(actions_in), int(bool(greedy))
        d.seed, d.counter_dev = int(seed) & 0xFFFFFFFFFFFFFFFF, _ptr(counter)
        d.actions_out, d.log_prob, d.entropy, d.logits_norm = _ptr(actions_out), _ptr(log_prob), _ptr(entropy), _ptr(logits_norm)
        self._ck(self.lib.vima_head_sample(self.h, C.byref(d), c_void_p(self._s())), "head_sample")
