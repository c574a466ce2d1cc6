"""oracle/value_rules.py -- TEST INFRASTRUCTURE ONLY.

The library's per-element quantisation rules (include/b200ms.h, b200ms_pack_pages) restated as torch integer and table
operations, so that they run on the GPU over every float32 bit pattern.  None of them uses torch's own dtype casts to
round: bf16 is the round-to-nearest-even bit formula, int8 is torch.round (half-even) of the fp32 product, e4m3 is a
nearest-even search of the 127-entry value table.  tests/test_value_oracle_cpu.py shows that each equals the numpy
oracle (maxsim_oracle.py) on a 2^20-pattern sample and every special class.

Inputs are int32 tensors of float32 BIT PATTERNS (any device); outputs are the packed bytes the library writes.
"""
from __future__ import annotations

import torch

from .maxsim_oracle import _E4M3

_E4M3_T = {}


def _table(device) -> torch.Tensor:
    key = str(device)
    if key not in _E4M3_T:
        _E4M3_T[key] = torch.as_tensor(_E4M3, dtype=torch.float64, device=device)
    return _E4M3_T[key]


def is_nan_bits(bits: torch.Tensor) -> torch.Tensor:
    return (bits & 0x7FFFFFFF) > 0x7F800000


def bf16_bits(bits: torch.Tensor) -> torch.Tensor:
    """float32 patterns -> bf16 patterns (int64 in 0..0xffff): RNE, overflow to +-inf, NaN -> 0x7fff."""
    u = bits.to(torch.int64) & 0xFFFFFFFF
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) & 0xFFFF
    return torch.where(is_nan_bits(bits), torch.full_like(r, 0x7FFF), r)


def int8_codes(bits: torch.Tensor, scale: float) -> torch.Tensor:
    """float32 patterns -> int8: round-half-even of the fp32 product, clamped to [-127, 127], NaN -> 0."""
    y = bits.view(torch.float32) * torch.tensor(scale, dtype=torch.float32, device=bits.device)
    r = torch.round(y).clamp(-127.0, 127.0)
    return torch.where(torch.isnan(y), torch.zeros_like(r), r).to(torch.int8)


def e4m3_codes(bits: torch.Tensor, scale: float) -> torch.Tensor:
    """float32 patterns -> e4m3 codes (uint8) of the fp32 product: nearest-even on the value table, saturating at 448,
    sign from the product's sign bit, NaN -> 0x7f."""
    y = bits.view(torch.float32) * torch.tensor(scale, dtype=torch.float32, device=bits.device)
    nan = torch.isnan(y)
    a = y.abs().to(torch.float64).clamp(max=448.0)
    a = torch.where(nan, torch.zeros_like(a), a)
    tab = _table(bits.device)
    hi = torch.searchsorted(tab, a, side="left").clamp(0, tab.numel() - 1)
    lo = (hi - 1).clamp(min=0)
    d_lo, d_hi = a - tab[lo], tab[hi] - a
    pick_hi = (d_hi < d_lo) | ((d_hi == d_lo) & (hi % 2 == 0))
    code = torch.where(pick_hi, hi, lo) | ((y.view(torch.int32) < 0).to(torch.int64) << 7)
    return torch.where(nan, torch.full_like(code, 0x7F), code).to(torch.uint8)


_BIT_WEIGHTS = {}


def sign_bytes(bits: torch.Tensor) -> torch.Tensor:
    """[rows, 128] float32 patterns -> [rows, 16] bytes: bit = x > 0 (so +-0 and NaN -> 0), MSB first."""
    key = str(bits.device)
    if key not in _BIT_WEIGHTS:
        _BIT_WEIGHTS[key] = torch.tensor([128, 64, 32, 16, 8, 4, 2, 1], dtype=torch.int32, device=bits.device)
    pos = (bits.view(torch.float32) > 0).view(-1, 16, 8).to(torch.int32)
    return (pos * _BIT_WEIGHTS[key]).sum(dim=-1).to(torch.uint8)


def packed_bytes(dtype: str, bits: torch.Tensor, scale: float = 1.0) -> torch.Tensor:
    """[rows, 128] float32 patterns -> [rows, row_bytes] uint8, the row layout of corpus dtype `dtype`."""
    rows = bits.view(-1, 128)
    if dtype == "bf16":
        b = bf16_bits(rows)
        return torch.stack([b & 0xFF, b >> 8], dim=-1).to(torch.uint8).view(rows.shape[0], 256)
    if dtype == "int8":
        return int8_codes(rows, scale).view(torch.uint8)
    if dtype == "fp8":
        return e4m3_codes(rows, scale)
    if dtype == "binary":
        return sign_bytes(rows)
    raise ValueError(dtype)
