"""The salt sampler of zero-knowledge commitments (plonky2_b200/csrc/gl_chacha.cuh) on the CPU: the numpy restatement
(tests/chacha_ref.py) against the public test vectors of RFC 8439, then the header's own source compiled for the host
against the restatement -- the sampling rule, the kernels' per-thread bodies and the leaf order of the salt fill, with
the default acceptance bound p and with a lowered bound under which about half of the words fall back to later
attempts."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import chacha_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RFC_KEY = bytes(range(32))
LOW_BOUND = 1 << 63     # ~ p / 2: about half of the words are rejected


def _bitrev(x, bits):
    return int(format(x, "0%db" % bits)[::-1], 2) if bits else 0


def test_rfc8439_block_function_vector():
    """RFC 8439 section 2.3.2: key 00..1f, nonce 00:00:00:09:00:00:00:4a:00:00:00:00, block count 1."""
    nonce = bytes.fromhex("000000090000004a00000000")
    n = [int.from_bytes(nonce[4 * j:4 * j + 4], "little") for j in range(3)]
    got = R.chacha20_blocks(RFC_KEY, [1], *n)[0]
    want = [0xe4e7f110, 0x15593bd1, 0x1fdd0f50, 0xc47120a3, 0xc7f4d1c7, 0x0368c033, 0x9aaa2204, 0x4e6cd4c3,
            0x466482d2, 0x09aa9f07, 0x05d7c214, 0xa2028bd9, 0xd19c12b5, 0xb94e16de, 0xe883d0cb, 0x4e3c50a2]
    assert [int(v) for v in got] == want
    assert got.astype("<u4").tobytes() == bytes.fromhex(
        "10f1e7e4d13b5915500fdd1fa32071c4c7d1f4c733c068030422aa9ac3d46c4e"
        "d2826446079faa0914c2d705d98b02a2b5129cd1de164eb9cbd083e8a2503c4e")


def test_rfc8439_keystream_vector():
    """RFC 8439 section 2.4.2: the sunscreen plaintext encrypted from counter 1 under nonce 00:00:00:00:00:00:00:4a:..."""
    pt = (b"Ladies and Gentlemen of the class of '99: If I could offer you only one tip for the future, "
          b"sunscreen would be it.")
    ct = bytes.fromhex(
        "6e2e359a2568f98041ba0728dd0d6981e97e7aec1d4360c20a27afccfd9fae0b"
        "f91b65c5524733ab8f593dabcd62b3571639d624e65152ab8f530c359f0861d8"
        "07ca0dbf500d6a6156a38e088a22b65e52bc514d16ccf806818ce91ab7793736"
        "5af90bbf74a35be6b40b8eedf2785e42874d")
    ks = R.keystream(RFC_KEY, 1, bytes.fromhex("000000000000004a00000000"), len(pt))
    assert bytes(a ^ b for a, b in zip(pt, ks)) == ct


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    """The header compiled for the host, once per acceptance bound."""
    libs = {}
    d = tmp_path_factory.mktemp("chacha_emu")
    for bound in (R.P, LOW_BOUND):
        out = str(d / ("libchacha_emu_%x.so" % bound))
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-DGL_FORCE_32BIT_PATH", "-DGL_CHACHA_BOUND=%#xULL" % bound,
                               "-shared", "-fPIC", "-o", out, os.path.join(ROOT, "tests", "emu", "chacha_emu.cpp")])
        L = C.CDLL(out)
        L.emu_chacha_bound.restype = C.c_uint64
        L.emu_chacha_block.argtypes = [C.c_char_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]
        L.emu_chacha_elements.argtypes = [C.c_char_p, C.c_uint32, C.c_uint64, C.c_uint64, C.c_void_p]
        L.emu_salt_fill.argtypes = [C.c_char_p, C.c_uint32, C.c_uint64, C.c_uint64, C.c_void_p]
        assert L.emu_chacha_bound() == bound
        libs[bound] = L
    return libs


def _keys():
    rng = np.random.default_rng(0xC4AC4A)
    return [RFC_KEY, bytes(32), bytes([0xFF] * 32)] + [rng.bytes(32) for _ in range(3)]


def _emu_elements(L, key, column, first, count):
    out = np.empty(count, dtype=np.uint64)
    assert L.emu_chacha_elements(key, column, first, count, out.ctypes.data) == 0   # block body == per-position rule
    return out


def test_header_block_function_on_host(emu):
    out = np.empty(16, dtype=np.uint32)
    for key in _keys()[:3]:
        for counter, n in ((1, (0x09000000, 0x4a000000, 0)), (0xFFFFFFFF, (3, 7, 0)), (0, (0, 0, 0))):
            emu[R.P].emu_chacha_block(key, counter, *n, out.ctypes.data)
            assert np.array_equal(out, R.chacha20_blocks(key, [counter], *n)[0])


@pytest.mark.parametrize("bound", [R.P, LOW_BOUND], ids=["p", "lowered"])
def test_header_sampler_on_host_matches_restatement(emu, bound):
    """2^16 elements in all: every key x column (0..3 and a large one) x (first, count) with unaligned starts and
    lengths, including positions near the end of the 2^35 range; every element canonical and below the bound."""
    L = emu[bound]
    total = 0
    cases = [(0, 1), (0, 8), (3, 5), (7, 9), (1, 1000), (12345, 2048), ((1 << 35) - 1000, 1000), ((1 << 20) + 5, 259)]
    for key in _keys():
        for column in (0, 1, 2, 3, 0xDEADBEEF):
            for first, count in cases:
                got = _emu_elements(L, key, column, first, count)
                want = R.samples(key, column, first, count, bound)
                assert np.array_equal(got, want), (key.hex(), column, first, count)
                assert (got < np.uint64(bound)).all()
                total += count
    assert total >= 1 << 16
    if bound == LOW_BOUND:   # the fallback really ran: about half of the attempt-0 words were rejected
        raw = R._words(_keys()[3], 0, 0, 0, 512).reshape(-1)
        assert 0.4 < float((raw >= np.uint64(bound)).mean()) < 0.6


@pytest.mark.parametrize("bound", [R.P, LOW_BOUND], ids=["p", "lowered"])
def test_header_salt_fill_on_host_leaf_order_and_shards(emu, bound):
    """k_chacha_salt's body: salt column s at leaf j = element (s, bitrev(j)), for every LDE size from 1 to 2^12 rows;
    each row-block shard (G up to 16) writes exactly its own leaves."""
    L = emu[bound]
    key = _keys()[4]
    for log_N in range(0, 13):
        N = 1 << log_N
        salt = R.salt_array(key, N, bound)
        want = salt[:, [_bitrev(j, log_N) for j in range(N)]]
        for G in (1, 2, 4, 8, 16):
            if G > N:
                continue
            got = np.concatenate([_fill(L, key, log_N, g * (N // G), N // G) for g in range(G)], axis=1)
            assert np.array_equal(got, want), (log_N, G)


def _fill(L, key, log_N, leaf0, nloc):
    out = np.full((4, nloc), 0xA5A5A5A5A5A5A5A5, dtype=np.uint64)
    L.emu_salt_fill(key, log_N, leaf0, nloc, out.ctypes.data)
    return out
