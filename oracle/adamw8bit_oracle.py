"""Reference of AdamW with blockwise 8-bit moments (torch on the CPU, fp32), the update rlaifv_adamw8bit_step computes.

State of a slice of n elements: fp32 master, uint8 codes code_m / code_v [n], fp32 absmax_m / absmax_v per block of
256 elements counted from the slice's first element (the last block may be partial). One step:
  1. m = map_m[code_m] * absmax_m, v = map_v[code_v] * absmax_v (the maps of zero2.dynamic_map);
  2. torch.optim.AdamW's arithmetic in adamw_elem's order (rowops.cu), weight decay on elements [0, decay_n);
  3. absmax_m = max|m|, absmax_v = max v per block over the new fp32 moments;
  4. each element's code is the index of the map entry nearest to m / absmax_m (v / absmax_v), ties to the lower
     index; a zero absmax stores the code of 0.
Every operation is one fp32 rounding, as the kernel's are when the compiler contracts nothing; with beta1 = beta2 = 0
the new moments are g and g * g under any contraction, so codes and absmax are then bit-exact.
"""
import numpy as np
import torch

from rlaifv_b200.zero2 import QBLOCK, dynamic_map

_F32 = torch.float32


def maps():
    return dynamic_map(True), dynamic_map(False)


def quantize(x, qmap):
    """Codes (int64) of the map entries nearest to x (fp32, normalised), ties to the lower index: the last entry <= x
    (entry 0 if none), then one compare with its upper neighbour."""
    i = (torch.searchsorted(qmap, x, right=True) - 1).clamp(0, qmap.numel() - 2)
    lo, hi = qmap[i], qmap[i + 1]
    return i + ((hi - x) < (x - lo)).to(torch.int64)


def block_absmax(x, n):
    """Per-block max of x ([n] fp32, already non-negative) over blocks of QBLOCK, the last one partial."""
    nb = (n + QBLOCK - 1) // QBLOCK
    pad = torch.zeros(nb * QBLOCK, dtype=_F32)
    pad[:n] = x
    return pad.view(nb, QBLOCK).amax(1)


def quantize_blocks(x, absmax, qmap):
    """Codes of x ([n]) in blocks whose scales are absmax ([nb]): x / absmax, 0 where absmax is 0."""
    n = x.numel()
    scale = absmax.repeat_interleave(QBLOCK)[:n]
    xn = torch.where(scale > 0, x / torch.where(scale > 0, scale, torch.ones_like(scale)), torch.zeros_like(x))
    return quantize(xn, qmap).to(torch.uint8)


def dequantize(codes, absmax, qmap):
    n = codes.numel()
    return qmap[codes.long()] * absmax.repeat_interleave(QBLOCK)[:n]


def step(master, code_m, code_v, absmax_m, absmax_v, grad, decay_n, lr, beta1, beta2, eps, weight_decay, step_no):
    """One update of a slice; returns (master, code_m, code_v, absmax_m, absmax_v, m, v, param_bf16) with m, v the fp32
    moments the step used. grad: bf16 or fp32 [n]."""
    map_m, map_v = maps()
    n = master.numel()
    f = np.float32
    g = grad.to(_F32)
    m = dequantize(code_m, absmax_m, map_m)
    v = dequantize(code_v, absmax_v, map_v)
    bc1 = f(1) - f(np.power(f(beta1), f(step_no)))
    bc2_sqrt = np.sqrt(f(1) - f(np.power(f(beta2), f(step_no))))
    keep = torch.full((n,), float(f(1) - f(lr) * f(weight_decay)), dtype=_F32)
    keep[decay_n:] = 1.0
    p = master.to(_F32) * keep
    m = float(f(beta1)) * m + float(f(1) - f(beta1)) * g
    v = float(f(beta2)) * v + (float(f(1) - f(beta2)) * g) * g
    denom = torch.sqrt(v) / float(bc2_sqrt) + float(f(eps))
    p = p - float(f(lr) / bc1) * (m / denom)
    am, av = block_absmax(m.abs(), n), block_absmax(v, n)
    return (p, quantize_blocks(m, am, map_m), quantize_blocks(v, av, map_v), am, av, m, v, p.to(torch.bfloat16))
