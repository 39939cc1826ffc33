"""Test infrastructure: a restatement of the device salt sampler in numpy -- the ChaCha20 block function of RFC 8439
section 2.3 and the sampling rule of plonky2_b200/csrc/gl_chacha.cuh -- written from the RFC and the documented rule,
not from the CUDA source:

    element (s, i) = the first word below the bound among  word (i mod 8) of block (i / 8) of the stream with
                     nonce (s, a, 0),  a = 0, 1, 2, ...

A keyed commitment's salt array (4 x N, by LDE row) is salt_array(key, N)."""
import numpy as np

P = 0xFFFFFFFF00000001
SIGMA = (0x61707865, 0x3320646E, 0x79622D32, 0x6B206574)   # "expand 32-byte k"


def key_words(key):
    assert len(key) == 32
    return [int.from_bytes(key[4 * j:4 * j + 4], "little") for j in range(8)]


def _rotl(x, r):
    return (x << np.uint32(r)) | (x >> np.uint32(32 - r))


def chacha20_blocks(key, counters, n0, n1, n2):
    """The block function for every counter: (len(counters), 16) uint32 serialised state words."""
    counters = np.asarray(counters, dtype=np.uint32)
    m = len(counters)
    init = [np.full(m, w, dtype=np.uint32) for w in SIGMA + tuple(key_words(key))]
    init += [counters.copy()] + [np.full(m, int(v) & 0xFFFFFFFF, dtype=np.uint32) for v in (n0, n1, n2)]
    x = [v.copy() for v in init]

    def qr(a, b, c, d):
        x[a] += x[b]
        x[d] = _rotl(x[d] ^ x[a], 16)
        x[c] += x[d]
        x[b] = _rotl(x[b] ^ x[c], 12)
        x[a] += x[b]
        x[d] = _rotl(x[d] ^ x[a], 8)
        x[c] += x[d]
        x[b] = _rotl(x[b] ^ x[c], 7)

    for _ in range(10):
        qr(0, 4, 8, 12), qr(1, 5, 9, 13), qr(2, 6, 10, 14), qr(3, 7, 11, 15)
        qr(0, 5, 10, 15), qr(1, 6, 11, 12), qr(2, 7, 8, 13), qr(3, 4, 9, 14)
    return np.stack([x[j] + init[j] for j in range(16)], axis=1)


def keystream(key, counter, nonce12, nbytes):
    """RFC 8439 section 2.4's keystream from a 12-byte nonce and an initial counter."""
    n = [int.from_bytes(nonce12[4 * j:4 * j + 4], "little") for j in range(3)]
    blocks = chacha20_blocks(key, np.arange(counter, counter + (nbytes + 63) // 64), *n)
    return blocks.astype("<u4").tobytes()[:nbytes]


def _words(key, column, attempt, blk0, nblocks):
    """The u64 words of blocks [blk0, blk0 + nblocks) of stream (column, attempt), in position order."""
    b = chacha20_blocks(key, np.arange(blk0, blk0 + nblocks, dtype=np.uint64).astype(np.uint32), column, attempt, 0)
    return b.astype(np.uint64)[:, 0::2] | (b.astype(np.uint64)[:, 1::2] << np.uint64(32))


def samples(key, column, first, count, bound=P, chunk_blocks=1 << 18):
    """Elements (column, first .. first + count - 1)."""
    out = np.empty(count, dtype=np.uint64)
    pos, done = first, 0
    while done < count:
        blk0 = pos >> 3
        nb = min(chunk_blocks, ((first + count - 1) >> 3) - blk0 + 1)
        w = _words(key, column, 0, blk0, nb).reshape(-1)[pos - 8 * blk0:]
        take = min(len(w), count - done)
        out[done:done + take] = w[:take]
        pos += take
        done += take
    bad, a = np.nonzero(out >= np.uint64(bound))[0], 1      # later attempts for the rejected positions
    while len(bad):
        p = np.uint64(first) + bad.astype(np.uint64)
        b = chacha20_blocks(key, (p >> np.uint64(3)).astype(np.uint32), column, a, 0).astype(np.uint64)
        k, rows = (p & np.uint64(7)).astype(np.int64), np.arange(len(bad))
        w = b[rows, 2 * k] | (b[rows, 2 * k + 1] << np.uint64(32))
        ok = w < np.uint64(bound)
        out[bad[ok]] = w[ok]
        bad, a = bad[~ok], a + 1
    return out


def salt_array(key, N, bound=P):
    """The salt (4 x N, salt[s][i] = element (s, i)) that a keyed commitment of N LDE rows draws."""
    return np.stack([samples(key, s, 0, N, bound) for s in range(4)])
