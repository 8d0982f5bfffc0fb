"""Per-launch timing of an Engine (CUDA events on the launching stream) with the algorithmic FLOPs / bytes of every
launch, for the roofline numbers bench.py reports."""
from __future__ import annotations

import ctypes as C

from . import _lib
from .tensors import _stream


def describe_ops(engine):
    out = []
    for o in engine.op_list:
        if o.kind == _lib.OP_CONV:
            d = o.conv
            ho, wo = d.h // d.stride, d.w // d.stride
            flops = 2.0 * d.n * ho * wo * d.c_out * d.c_in * d.ksize * d.ksize
            out_b = d.n * ho * wo * d.c_out * (4 if d.out_f32 else 2) * (4 if d.upsample else 1)
            byts = d.n * d.h * d.w * d.c_in * 2 + out_b + d.c_out * d.c_in * d.ksize**2 * 2 + (out_b if d.res else 0)
            out.append(dict(kind="conv_tc", shape=f"{d.c_in}->{d.c_out} k{d.ksize} s{d.stride} @{d.h}x{d.w} n{d.n}"
                            + (" +res" if d.res else "") + (" +up2x" if d.upsample else "") + (" head" if d.out_f32 else ""),
                            flops=flops, bytes=byts))
        elif o.kind == _lib.OP_CONV_FIRST:
            d = o.first
            flops = 2.0 * d.n * d.h * d.w * d.c_out * 27
            byts = d.n * d.h * d.w * (3 * (1 if d.in_dtype == _lib.IN_U8 else 4) + d.c_out * 2)
            out.append(dict(kind="conv_first", shape=f"3->{d.c_out} k3 s1 @{d.h}x{d.w} n{d.n}", flops=flops, bytes=byts))
        elif o.kind == _lib.OP_MAXPOOL:
            d = o.pool
            byts = d.n * d.c * 2 * (d.h * d.w + d.ho * d.wo)
            out.append(dict(kind="maxpool", shape=f"c{d.c} k{d.k} s{d.stride} @{d.h}x{d.w} n{d.n}", flops=0.0, bytes=byts))
        elif o.kind == _lib.OP_DECODE:
            d = o.decode
            rows = sum(d.na * d.levels[i].ny * d.levels[i].nx for i in range(d.nl))
            out.append(dict(kind="decode", shape=f"rows {rows} no {d.no} n{d.bs}", flops=0.0,
                            bytes=d.bs * rows * d.no * (12 if any(d.levels[l].raw_out for l in range(d.nl)) else 8)))
    return out


def time_ops(engine, x=None, iters=5):
    """Returns [{kind, shape, flops, bytes, ms, tflops, gbs}] for one forward (average over ``iters`` passes)."""
    n = engine.n_ops
    ms = (C.c_float * n)()
    _lib.check(_lib.lib().y3_model_forward_timed(engine.handle, x.data_ptr() if x is not None else None, _stream(), ms, iters),
               "y3_model_forward_timed")
    ops = describe_ops(engine)
    for o, t in zip(ops, ms):
        o["ms"] = float(t)
        o["tflops"] = o["flops"] / (t * 1e9) if t > 0 else 0.0
        o["gbs"] = o["bytes"] / (t * 1e6) if t > 0 else 0.0
    return ops
