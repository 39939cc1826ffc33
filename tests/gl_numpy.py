"""Exact Goldilocks arithmetic on numpy uint64 arrays, vectorised: a reference for device columns of 2^24 rows and more,
where per-element Python integers take minutes. Test infrastructure only.

Every operation accepts any u64 word (canonical or not) and returns canonical values in [0, p). mul forms the exact
128-bit product from 32-bit limbs and reduces it with 2^64 = 2^32 - 1 and 2^96 = -1 (mod p). Nothing here inverts:
the tests pin device columns with identities that only multiply. The arithmetic is checked against Python integers in
tests/test_gpu_stark_large.py."""
import os

import numpy as np

P = 0xFFFFFFFF00000001
_P = np.uint64(P)
_EPS = np.uint64(0xFFFFFFFF)                 # 2^64 - p = 2^32 - 1
_M32 = np.uint64(0xFFFFFFFF)
_S32 = np.uint64(32)
W = 7                                        # F_{p^2} = F_p[X] / (X^2 - 7)
_PAR_MIN = 1 << 18
_THREADS = min(16, os.cpu_count() or 1)


def u64(a):
    return np.asarray(a, dtype=np.uint64)


def canon(a):
    a = u64(a)
    return np.where(a >= _P, a - _P, a)


def add(a, b):
    return _threaded(_add, u64(a), u64(b))


def _add(a, b):
    a, b = canon(a), canon(b)
    with np.errstate(over="ignore"):
        s = a + b
        s = np.where(s < a, s + _EPS, s)     # a carry out of 2^64 is worth 2^32 - 1; s + 2^32 - 1 < p then
    return canon(s)


def sub(a, b):
    return _threaded(_sub, u64(a), u64(b))


def _sub(a, b):
    a, b = canon(a), canon(b)
    with np.errstate(over="ignore"):
        return np.where(a >= b, a - b, a - b + _P)


def neg(a):
    return sub(np.uint64(0), a)


def _threaded(fn, a, b):
    """fn(a, b) over row blocks on a thread pool (numpy releases the GIL in its loops): a and b are arrays of one shape
    or scalars. Small or other operands run in one call."""
    shape = np.broadcast_shapes(a.shape, b.shape)
    n = int(np.prod(shape))
    if n < _PAR_MIN or any(x.shape not in ((), shape) for x in (a, b)):
        return fn(a, b)
    from concurrent.futures import ThreadPoolExecutor

    out = np.empty(n, dtype=np.uint64)
    flat = [x if x.ndim == 0 else x.reshape(-1) for x in (a, b)]
    step = -(-n // _THREADS)

    def block(s):
        out[s:s + step] = fn(*[x if x.ndim == 0 else x[s:s + step] for x in flat])

    with ThreadPoolExecutor(_THREADS) as pool:
        list(pool.map(block, range(0, n, step)))
    return out.reshape(shape)


def mul(a, b):
    return _threaded(_mul, u64(a), u64(b))


def _mul(a, b):
    with np.errstate(over="ignore"):
        a0, a1 = a & _M32, a >> _S32
        b0, b1 = b & _M32, b >> _S32
        p00, p01, p10, p11 = a0 * b0, a0 * b1, a1 * b0, a1 * b1   # each < 2^64
        mid = p01 + p10
        mid_carry = (mid < p01).astype(np.uint64)                  # worth 2^96 = 2^32 in the high word
        lo = p00 + (mid << _S32)
        lo_carry = (lo < p00).astype(np.uint64)
        hi = p11 + (mid >> _S32) + (mid_carry << _S32) + lo_carry  # the product is hi * 2^64 + lo < 2^128
        # hi * 2^64 + lo = hl * 2^64 + hh * 2^96 + lo = lo + hl * (2^32 - 1) - hh  (mod p)
        hl, hh = hi & _M32, hi >> _S32
        t0 = lo - hh
        t0 = np.where(lo < hh, t0 - _EPS, t0)                    # borrow: t0 + 2^64 = t0 - (2^32 - 1) mod p
        t1 = hl * _EPS
        t2 = t0 + t1
        t2 = np.where(t2 < t1, t2 + _EPS, t2)
    return canon(t2)


def square(a):
    return mul(a, a)


def pow_scalar(base, e):
    """base^e for a Python integer e >= 0, elementwise by square-and-multiply."""
    out = np.ones_like(u64(base))
    sq = canon(base)
    while e:
        if e & 1:
            out = mul(out, sq)
        sq = mul(sq, sq)
        e >>= 1
    return out


def powers(base, n):
    """[1, base, base^2, ..., base^(n-1)] for a scalar base, by doubling: the filled prefix times base^len."""
    out = np.empty(n, dtype=np.uint64)
    if n == 0:
        return out
    out[0] = 1
    filled, step = 1, canon(np.uint64(int(base) % 2**64))
    while filled < n:
        take = min(filled, n - filled)
        out[filled:filled + take] = mul(out[:take], step)
        filled += take
        step = mul(step, step)
    return out


def ext_mul(a, b):
    """(a0 + a1 X)(b0 + b1 X) mod X^2 - 7 on pairs (c0, c1) of arrays."""
    a0, a1 = a
    b0, b1 = b
    return add(mul(a0, b0), mul(np.uint64(W), mul(a1, b1))), add(mul(a0, b1), mul(a1, b0))


def brev(idx, bits):
    """Bit reversal of every index over `bits` bits."""
    idx = u64(idx)
    out = np.zeros_like(idx)
    for k in range(bits):
        out |= ((idx >> np.uint64(k)) & np.uint64(1)) << np.uint64(bits - 1 - k)
    return out
