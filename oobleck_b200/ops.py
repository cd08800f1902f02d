"""Thin tensor-level wrappers over the C ABI (torch supplies device memory and streams only)."""
from __future__ import annotations

import ctypes as C

import torch

from . import lib as L

NSPLIT_PARITY = 3  # fp32-grade split (6 tensor-core products); see csrc/common.cuh


def _ptr(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def new_planes(rows: int, cols: int, nplanes: int = 3, device="cuda") -> torch.Tensor:
    """bf16 [nplanes, rows, cols] split-plane buffer (cols must be a multiple of 8)."""
    assert cols % 8 == 0, cols
    return torch.empty((nplanes, rows, cols), dtype=torch.bfloat16, device=device)


def planes_desc(p: torch.Tensor, rows=None, cols=None, fp16: bool = False) -> L.Planes:
    """``fp16``: describe the fp16 pair (planes 3, 4) of a 5-plane buffer instead of its bf16 planes."""
    assert p.dtype == torch.bfloat16 and p.dim() == 3 and p.stride(2) == 1
    rows = rows if rows is not None else p.shape[1]
    cols = cols if cols is not None else p.shape[2]
    if fp16:
        assert p.shape[0] == L.planes_count(L.PLANES_BF16X3_FP16_PAIR)
        return L.Planes(p[3:].data_ptr(), rows, cols, p.stride(1), p.stride(0), 2, 1)
    return L.Planes(p.data_ptr(), rows, cols, p.stride(1), p.stride(0), min(p.shape[0], 3), 0)


def split(x: torch.Tensor, out: torch.Tensor | None = None, nplanes: int = 3) -> torch.Tensor:
    """fp32 [rows, cols] -> planes [planes_count(nplanes), rows, cols] (``nplanes``: plane-set code)."""
    x = x.contiguous()
    rows, cols = x.shape
    if out is None:
        out = new_planes(rows, cols, L.planes_count(nplanes), x.device)
    L.call("oob_split_planes", _ptr(x), _ptr(out), x.numel(), out.stride(0), nplanes, _stream())
    return out


def planes_to_float(p: torch.Tensor, fp16: bool = False) -> torch.Tensor:
    if fp16:   # planes 3, 4 hold fp16 bit patterns: x ~= h0 + 2^-11 h1
        h = p[3:5].view(torch.float16).float()
        return h[0] + h[1] / 2048.0
    return p[:3].float().sum(0)


def pair_to_float(p: torch.Tensor) -> torch.Tensor:
    """fp16 pair stored at planes 0, 1 (``OOB_PLANES_FP16_PAIR`` output of a gradient producer)."""
    h = p[0:2].view(torch.float16).float()
    return h[0] + h[1] / 2048.0


PLANES_FP16_PAIR = L.PLANES_FP16_PAIR


def gemm(a: torch.Tensor, a_mn: bool, b: torch.Tensor, b_mn: bool, M: int, N: int, K: int, *, nsplit=NSPLIT_PARITY,
         d=None, bias=None, resid=None, accumulate=False, act=L.ACT_NONE, aux=None, planes_out=None, alpha=1.0,
         a_fp16=False, b_fp16=False, planes_code=None, a_pair0=False, b_pair0=False):
    """``planes_code``: plane-set code of ``planes_out`` (default: its number of planes; PLANES_FP16_PAIR for a 2-plane
    pair-only buffer).  ``a_pair0`` / ``b_pair0``: the operand is a pair-only buffer (fp16 pair at planes 0, 1)."""
    e = L.GemmEpilogue()
    e.d = 0 if d is None else d.data_ptr()
    e.ldd = 0 if d is None else d.stride(0)
    e.bias = 0 if bias is None else bias.data_ptr()
    e.resid = 0 if resid is None else resid.data_ptr()
    e.ldr = 0 if resid is None else resid.stride(0)
    e.accumulate = int(accumulate)
    e.act = act
    e.aux = 0 if aux is None else aux.data_ptr()
    e.ldaux = 0 if aux is None else aux.stride(0)
    e.planes = 0 if planes_out is None else planes_out.data_ptr()
    e.ldp = 0 if planes_out is None else planes_out.stride(1)
    e.plane_stride = 0 if planes_out is None else planes_out.stride(0)
    e.nplanes_out = 0 if planes_out is None else (planes_out.shape[0] if planes_code is None else planes_code)
    e.alpha = alpha
    def desc(t, fp16, pair0):
        if pair0:
            return L.Planes(t.data_ptr(), t.shape[1], t.shape[2], t.stride(1), t.stride(0), 2, 1)
        return planes_desc(t, fp16=fp16)
    A, B = desc(a, a_fp16, a_pair0), desc(b, b_fp16, b_pair0)
    L.call("oob_gemm", C.byref(A), int(a_mn), C.byref(B), int(b_mn), M, N, K, nsplit, C.byref(e), _stream())
