"""ORACLE (test infrastructure only -- never imported by the product path's kernels).

The device stream of RandomVariable nodes (``aesara_b200/csrc/ab_random.cu``), restated in NumPy
uint64 arithmetic, and the RandomVariable handler of the program interpreter
(``oracle/program_np.py``), which importing this module installs.

The stream is not the reference's NumPy stream (its ziggurat normal consumes a data-dependent
number of raw draws); what is shared with the reference is the Generator handling of
RandomVariable.perform (aesara/tensor/random/op.py:344-374): draw from the rng itself when the Op
is in place, from a copy of it otherwise, and return that Generator.

``tests/`` and ``aesara_b200.debug.check_function`` (which checks a random variable's device
sample against this stream) import this module.
"""

import numpy as np

from .program_np import _h

_M32 = np.uint64(0xFFFFFFFF)
_PHILOX_M = (np.uint64(0xD2511F53), np.uint64(0xCD9E8D57))
_PHILOX_W = (np.uint64(0x9E3779B9), np.uint64(0xBB67AE85))
_PI = np.longdouble("3.14159265358979323846264338327950288")
_CHUNK_BLOCKS = 1 << 20


def philox4x32_10(counter, key):
    """Philox4x32-10 (Salmon et al., SC'11; Random123 constants): ``counter`` [..., 4] and
    ``key`` [2] of 32-bit words -> the 4 output words, as uint64 arrays holding 32-bit values."""
    counter = np.asarray(counter, dtype=np.uint64)
    c0, c1, c2, c3 = (counter[..., k] for k in range(4))
    k0, k1 = np.uint64(key[0]), np.uint64(key[1])
    for _ in range(10):
        p0 = _PHILOX_M[0] * c0  # 32 x 32 -> 64 bits, exact in uint64
        p1 = _PHILOX_M[1] * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _M32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _M32
        k0 = (k0 + _PHILOX_W[0]) & _M32
        k1 = (k1 + _PHILOX_W[1]) & _M32
    return np.stack([c0, c1, c2, c3], axis=-1)


def philox_words(key, first_block, n_blocks):
    """Words 4*first_block .. 4*(first_block+n_blocks)-1 of the stream of the 64-bit ``key``."""
    key = int(key)
    b = np.arange(first_block, first_block + n_blocks, dtype=np.uint64)
    z = np.zeros_like(b)
    ctr = np.stack([b & _M32, b >> np.uint64(32), z, z], axis=-1)
    return philox4x32_10(ctr, (key & 0xFFFFFFFF, key >> 32)).reshape(-1)


def _unit24(w):
    return (w >> np.uint64(8)).astype(np.float64) * 2.0 ** -24


def _bits53(lo, hi):
    return ((hi << np.uint64(32)) | lo) >> np.uint64(11)


def random_raw(dist, dtype, key, n):
    """Per element, the value before the parameters: the uniform in [0, 1) (float64, exact),
    or for ``normal`` the standard normal z computed in long double from the same words."""
    per = 2 if np.dtype(dtype) == np.float64 and dist != "bernoulli" else 4
    blocks = (n + per - 1) // per
    out = np.empty(blocks * per, dtype=np.longdouble if dist == "normal" else np.float64)
    for b0 in range(0, blocks, _CHUNK_BLOCKS):
        nb = min(_CHUNK_BLOCKS, blocks - b0)
        w = philox_words(key, b0, nb)
        if dist == "normal":
            if per == 4:  # pair m: words 2m, 2m+1
                a, c = w[0::2], w[1::2]
                u1 = ((a >> np.uint64(8)) + np.uint64(1)).astype(np.longdouble) * np.longdouble(2.0 ** -24)
                u2 = _unit24(c).astype(np.longdouble)
            else:  # pair m: words 4m..4m+3
                u1 = (_bits53(w[0::4], w[1::4]) + np.uint64(1)).astype(np.longdouble) * np.longdouble(2.0 ** -53)
                u2 = _bits53(w[2::4], w[3::4]).astype(np.longdouble) * np.longdouble(2.0 ** -53)
            r = np.sqrt(-2 * np.log(u1))
            z = np.empty(2 * r.size, dtype=np.longdouble)
            z[0::2] = r * np.cos(2 * _PI * u2)
            z[1::2] = r * np.sin(2 * _PI * u2)
            v = z
        elif per == 4:
            v = _unit24(w)
        else:
            v = _bits53(w[0::2], w[1::2]).astype(np.float64) * 2.0 ** -53
        out[b0 * per:(b0 + nb) * per] = v
    return out[:n]


def random_sample(dist, dtype, key, shape, params):
    """The device's sample of ``shape`` for the 64-bit ``key``: uniform and Bernoulli draws bit
    for bit; for ``normal`` the truth ``loc + scale * z`` in float64 from long-double z (the
    device computes in ``dtype`` and is compared within a tolerance)."""
    shape = tuple(int(s) for s in shape)
    n = int(np.prod(shape)) if shape else 1
    pdt = np.float64 if dist == "bernoulli" else np.dtype(dtype)
    ps = [np.broadcast_to(np.asarray(p).astype(pdt), shape).reshape(-1) for p in params]
    check_random_params(dist, ps)
    raw = random_raw(dist, dtype, key, n)
    if dist == "uniform":
        lo, hi = ps
        u = raw.astype(pdt)  # exact: 24 or 53 significant bits
        with np.errstate(all="ignore"):
            out = lo + (hi - lo) * u  # one rounding per operation, in the output dtype
    elif dist == "normal":
        loc, scale = (p.astype(np.float64) for p in ps)
        with np.errstate(all="ignore"):
            out = (loc + scale * raw).astype(np.float64)
    else:
        out = (raw < ps[0]).astype(np.int64)
    return out.reshape(shape)


def check_random_params(dist, ps):
    """The ValueErrors NumPy / SciPy raise for these parameters."""
    if dist == "normal" and np.any(ps[1] < 0):
        raise ValueError("scale < 0")
    if dist == "bernoulli" and not np.all((ps[0] >= 0) & (ps[0] <= 1)):
        raise ValueError("p < 0, p > 1 or p is NaN")


def random_shape(size, params):
    """Output shape of a RandomVariable node: ``size`` if given, else the broadcast parameter
    shape; the parameters must broadcast to it (NumPy's rule)."""
    size = tuple(int(s) for s in np.asarray(size).reshape(-1))
    pshapes = [np.shape(p) for p in params]
    shape = size if size else tuple(np.broadcast_shapes(*pshapes))
    try:
        full = tuple(np.broadcast_shapes(shape, *pshapes))
    except ValueError:
        full = None
    if full != shape:
        raise ValueError(f"shape mismatch: parameters of shapes {pshapes} cannot be broadcast to size {shape}")
    return shape


@_h("RandomVariable")
def _random_variable(node, args, prog):  # aesara/tensor/random/op.py:344 (perform)
    import copy

    p = node.params
    rng, size, _dtype, *params = args
    params = params[-1:] if p["dist"] == "bernoulli" else params
    if not p["inplace"]:
        rng = copy.copy(rng)
    key = int(rng.integers(0, 2 ** 64, dtype=np.uint64))
    shape = random_shape(size, params)
    return [rng, random_sample(p["dist"], p["dtype"], key, shape, params)]
