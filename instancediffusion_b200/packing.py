"""Weight re-layouts done once at load time (host side; pure index permutations, no arithmetic)."""
from __future__ import annotations

from typing import Optional, Tuple

import torch


GEGLU_GROUP = 128  # rows per value / gate group of a packed GEGLU projection (csrc/gemm2.cu: BN = 256)


def pack_conv3x3(w: torch.Tensor) -> torch.Tensor:
    """(Cout, Cin, 3, 3) -> (Cout, 9*Cin) with k = (ky*3 + kx)*Cin + c: the K order in which the
    implicit-GEMM kernel walks the taps (csrc/gemm.cu)."""
    cout, cin, kh, kw = w.shape
    assert kh == 3 and kw == 3
    return w.permute(0, 2, 3, 1).reshape(cout, 9 * cin).contiguous()


def pack_conv3x3_taps(w: torch.Tensor) -> torch.Tensor:
    """(Cout, Cin, 3, 3) -> (9*Cin, Cout) with row k = (ky*3 + kx)*Cin + c: the layout of
    idiff_conv_in_select, whose threads each read a pair of output channels."""
    cout, cin, kh, kw = w.shape
    assert kh == 3 and kw == 3
    return w.permute(2, 3, 1, 0).reshape(9 * cin, cout).contiguous()


def pack_conv1x1(w: torch.Tensor) -> torch.Tensor:
    """(Cout, Cin, 1, 1) -> (Cout, Cin)."""
    return w.reshape(w.shape[0], w.shape[1]).contiguous()


def pack_geglu(w: torch.Tensor, bias: Optional[torch.Tensor]) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """GEGLU.proj (attention.py:39): rows [0, inner) are the value half and [inner, 2*inner) the
    gate half (chunk(2, dim=-1), :42).  Interleave them per GEGLU_GROUP = 128 so that one 256-column
    accumulator tile holds value columns [0,128) and their gates [128,256) -- the GEGLU epilogue then
    needs a single tile."""
    two_inner = w.shape[0]
    inner = two_inner // 2
    g = GEGLU_GROUP
    assert inner % g == 0, f"GEGLU inner dim must be a multiple of {g}"
    t = inner // g
    wv = w[:inner].reshape(t, g, -1)
    wg = w[inner:].reshape(t, g, -1)
    wp = torch.stack([wv, wg], dim=1).reshape(two_inner, -1).contiguous()
    bp = None
    if bias is not None:
        bv = bias[:inner].reshape(t, g)
        bg = bias[inner:].reshape(t, g)
        bp = torch.stack([bv, bg], dim=1).reshape(two_inner).contiguous()
    return wp, bp
