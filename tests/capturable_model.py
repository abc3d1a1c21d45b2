"""CPU model of the scalar block of a capturable FlatSGD / FlatAdamW (csrc/flat_scalars.cuh): the scalars of the update run
when the device step counter reads ``s`` (t = s + 1), in the kernel's order of explicitly rounded fp64 operations, each
result rounded once to fp32.  Python's float arithmetic and ``math.sqrt`` are IEEE round-to-nearest, as ``__dmul_rn``,
``__dadd_rn``, ``__ddiv_rn`` and ``__dsqrt_rn`` are."""
import math
import struct


def f32(x: float) -> float:
    return struct.unpack("f", struct.pack("f", x))[0]


def flat_pow(b: float, t: int) -> float:
    """``b ** t`` by squaring, the factors taken from the lowest bit of ``t`` up (flat_pow)."""
    r = 1.0
    while t:
        if t & 1:
            r = r * b
        b = b * b
        t >>= 1
    return r


def block(lr_t: float, wd: float, betas=(0.0, 0.0), eps: float = 0.0, s: int = 0, pow_fn=flat_pow) -> dict:
    """The block's values for one group: ``lr_t`` is the fp32 lr of the update (lr_schedule_lr), ``wd`` the group's fp64
    weight decay.  ``adamw`` is AdamwScalars' order: decay, w1, beta2, c2, step_size, sbc2, eps."""
    b1, b2 = betas
    t = s + 1
    p1, p2 = pow_fn(b1, t), pow_fn(b2, t)
    decay = f32(1.0 - lr_t * wd)
    step_size = f32(lr_t / (1.0 - p1))
    return {"lr": f32(lr_t), "wd": f32(wd), "decay": decay, "step_size": step_size,
            "adamw": [decay, f32(1.0 - b1), f32(b2), f32(1.0 - b2), step_size, f32(math.sqrt(1.0 - p2)), f32(eps)]}


def ulps(a: float, b: float) -> int:
    """Distance of two fp32 values in units in the last place (same sign)."""
    ia, ib = (struct.unpack("i", struct.pack("f", x))[0] for x in (a, b))
    return abs(ia - ib)
