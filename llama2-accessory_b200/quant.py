"""OmniQuant-style W{2,3,4}A16 weight quantisation and packing (host side of the C-ABI packer).

Takes the place of the weight half of accessory/util/quant.py:116-130 (bnb.nn.Params4bit).  The
uniform-affine quantiser follows the published OmniQuant algorithm with learned weight clipping off
(github.com/OpenGVLab/OmniQuant, quantize/quantizer.py::UniformAffineQuantizer; the reference only
links it from README.md:37):
    scale = clamp((max-min)/(2^b-1), 1e-5, 1e4);  zero = round(clamp(-min/scale, -1e4, 1e4))
    q = clamp(round(w/scale) + zero, 0, 2^b-1);   w_hat = fp16(fp16(q - zero) * fp16(scale))
"""
import ctypes as C
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from . import _cabi


def quantize_weight(w: torch.Tensor, bits: int, group_size: int = 0):
    """w [N,K] -> (q uint8 [N,K], scale fp16 [N,G], zero fp16 [N,G] integer valued, g)."""
    assert w.dim() == 2 and bits in (2, 3, 4)
    N, K = w.shape
    g = K if (not group_size or group_size <= 0 or group_size >= K) else int(group_size)
    if K % g:
        raise ValueError(f"K={K} is not a multiple of group_size={g}")
    G = K // g
    x = w.detach().float().reshape(N, G, g)
    lo, hi = x.amin(-1, keepdim=True), x.amax(-1, keepdim=True)
    qmax = float(2 ** bits - 1)
    # true IEEE division on every device: torch's CUDA `tensor / python_scalar` multiplies by the rounded
    # reciprocal, and a 1-ulp change of `scale` flips round(-lo/scale) whenever it sits at x.5 (symmetric weights)
    scale = ((hi - lo).double() / qmax).float().clamp(1e-5, 1e4)
    zero = (-lo / scale).clamp(-1e4, 1e4).round()
    if float(zero.abs().max()) > 1024:
        raise ValueError("degenerate group: |zero point| > 1024 is not representable in the packed format")
    q = (torch.round(x / scale) + zero).clamp(0.0, qmax)
    return (q.to(torch.uint8).reshape(N, K), scale.to(torch.float16).reshape(N, G),
            zero.to(torch.float16).reshape(N, G), g)


def dequantize(q, scale, zero, group_size):
    """fp16(fp16(q - z) * s16): the fake-quantised weight the reference model is given."""
    N, K = q.shape
    G = K // group_size
    d = (q.reshape(N, G, group_size).float() - zero.reshape(N, G, 1).float()).to(torch.float16)
    return (d * scale.reshape(N, G, 1)).to(torch.float16).reshape(N, K)


@dataclass
class PackedLinear:
    """A linear layer shard in the engine's packed device format (include/b200_decode.h b200_linear_t)."""
    bits: int
    N: int
    K: int
    group_size: int  # 0 = per output channel
    qweight: torch.Tensor            # uint8, packed
    scales: Optional[torch.Tensor]   # uint8 view of half2 (s, z); None for fp16 weights

    def c_struct(self) -> _cabi.Linear:
        return _cabi.Linear(self.bits, self.N, self.K, self.group_size, self.qweight.data_ptr(),
                            self.scales.data_ptr() if self.scales is not None else None)

    @property
    def nbytes(self) -> int:
        return self.qweight.numel() + (self.scales.numel() if self.scales is not None else 0)


def container_bits(bits: int, group_size: int, K: int) -> int:
    """Storage codec actually used.  W3 with group scales and W2 with 64-wide groups do not align with
    their codecs' k-blocks (80 / 128), so they are stored in the 4-bit container (DESIGN.md)."""
    grouped = bool(group_size) and 0 < group_size < K
    if bits == 3 and grouped:
        return 4
    if bits == 2 and grouped and group_size != 128:
        return 4
    return bits


def _np_ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


def pack_quantized(q: torch.Tensor, scale: torch.Tensor, zero: torch.Tensor, bits: int, group_size: int,
                   device) -> PackedLinear:
    """(q uint8 [N,K], scale/zero fp16 [N,G]) -> PackedLinear on `device` (packing runs on the host).

    Zero points must be integers with |z| <= 1024: the kernels dequantise (1024 + q) - (1024 + z) in fp16, which is exact
    only in that range, and a fractional z would round silently."""
    zf = zero.detach().float()
    if zf.numel() and (not torch.equal(zf, zf.round()) or float(zf.abs().max()) > 1024):
        raise ValueError("zero points must be integers with |z| <= 1024 in the packed format")
    lib = _cabi.lib()
    N, K = q.shape
    gs = 0 if (not group_size or group_size >= K) else int(group_size)
    cb = container_bits(bits, gs, K)
    qn = np.ascontiguousarray(q.detach().cpu().numpy().astype(np.uint8))
    out = np.empty(lib.b200_packed_weight_bytes(cb, N, K), dtype=np.uint8)
    _cabi.check(lib.b200_pack_weight(cb, N, K, _np_ptr(qn), _np_ptr(out)), "b200_pack_weight")
    sn = np.ascontiguousarray(scale.detach().cpu().contiguous().view(torch.int16).numpy().astype(np.uint16))
    zn = np.ascontiguousarray(zero.detach().cpu().contiguous().view(torch.int16).numpy().astype(np.uint16))
    so = np.empty(lib.b200_packed_scale_bytes(N, K, gs), dtype=np.uint8)
    _cabi.check(lib.b200_pack_scales(N, K, gs, _np_ptr(sn), _np_ptr(zn), _np_ptr(so)), "b200_pack_scales")
    return PackedLinear(cb, N, K, gs, torch.from_numpy(out).to(device), torch.from_numpy(so).to(device))


def pack_fp16(w: torch.Tensor, device) -> PackedLinear:
    lib = _cabi.lib()
    N, K = w.shape
    wn = np.ascontiguousarray(w.detach().cpu().to(torch.float16).contiguous().view(torch.int16).numpy().astype(np.uint16))
    out = np.empty(N * K * 2, dtype=np.uint8)
    _cabi.check(lib.b200_pack_f16(N, K, _np_ptr(wn), _np_ptr(out)), "b200_pack_f16")
    return PackedLinear(16, N, K, 0, torch.from_numpy(out).to(device), None)


def unpack_quantized(pl: PackedLinear) -> torch.Tensor:
    lib = _cabi.lib()
    src = np.ascontiguousarray(pl.qweight.cpu().numpy())
    out = np.empty((pl.N, pl.K), dtype=np.uint8)
    _cabi.check(lib.b200_unpack_weight(pl.bits, pl.N, pl.K, _np_ptr(src), _np_ptr(out)), "b200_unpack_weight")
    return torch.from_numpy(out)


def random_packed(bits: int, N: int, K: int, group_size: int, device, seed: int = 0) -> PackedLinear:
    """Synthetic weights generated directly in packed form on the device (any bit pattern is a valid
    packed weight).  scale ~ 2/((2^b-1) sqrt(K)), zero = 2^(b-1): weights ~ U(-1/sqrt(K), 1/sqrt(K))."""
    lib = _cabi.lib()
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    gs = 0 if (not group_size or group_size >= K) else int(group_size)
    cb = container_bits(bits, gs, K)
    nb = lib.b200_packed_weight_bytes(cb, N, K)
    qw = torch.randint(0, 256, (nb,), dtype=torch.uint8, device=device, generator=g)
    if cb == 16:
        w = ((torch.rand((nb // 2,), device=device, generator=g) * 2 - 1) / (K ** 0.5)).to(torch.float16)
        return PackedLinear(16, N, K, 0, w.view(torch.uint8), None)
    if cb != bits:  # a narrower code stored in the 4-bit container: keep fields < 2^bits
        m = (1 << bits) - 1
        qw = qw & ((m << 4) | m)
    G = 1 if gs == 0 else K // gs
    s = (2.0 / ((2 ** bits - 1) * K ** 0.5)) * (0.75 + 0.5 * torch.rand((N * G,), device=device, generator=g))
    z = torch.full((N * G,), float(2 ** (bits - 1)), device=device)
    sz = torch.stack([s, z], dim=1).to(torch.float16).contiguous()
    return PackedLinear(cb, N, K, gs, qw, sz.view(torch.uint8).reshape(-1))
