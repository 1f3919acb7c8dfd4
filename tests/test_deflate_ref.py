"""CPU: the deflate references of tests/deflate_ref.py, pinned before the GPU encoder's tests rely on them --
inflate_blocks against zlib on stored, fixed and dynamic blocks and on corrupted streams, optimal_limited_cost against an
exhaustive search over every length vector that satisfies Kraft's inequality."""
import itertools
import zlib

import numpy as np
import pytest

from deflate_ref import (CL_ORDER, EOB, InflateError, at_least_two, dist_code, histograms, huffman_cost, inflate_blocks,
                         len_code, optimal_limited_cost, replay)


def _corpus():
    g = np.random.default_rng(7)
    text = b''.join(b'the quick brown fox %d jumps over the lazy dog %d\n' % (i, i * i % 97) for i in range(3000))
    noise = g.integers(0, 256, 40000, dtype=np.uint8).tobytes()
    skew = g.geometric(0.3, 60000).clip(0, 255).astype(np.uint8).tobytes()
    runs = bytes([0]) * 5000 + bytes(range(256)) * 20 + bytes([7]) * 70000
    far = noise[:20000] + skew[:12000] + noise[:20000]          # a repeat at distance 32000
    return {'text': text, 'noise': noise, 'skew': skew, 'runs': runs, 'far': far, 'empty': b'', 'one': b'x'}


CORPUS = _corpus()
SETTINGS = [('level', 0), ('level', 1), ('level', 6), ('level', 9),
            ('strategy', zlib.Z_HUFFMAN_ONLY), ('strategy', zlib.Z_RLE), ('strategy', zlib.Z_FIXED)]


def _compress(data, kind, v):
    if kind == 'level':
        return zlib.compress(data, v)
    c = zlib.compressobj(6, zlib.DEFLATED, 15, 8, v)
    return c.compress(data) + c.flush()


def _check_block(b):
    assert b.btype in (0, 1, 2)
    if b.btype == 0:
        assert not b.tokens and len(b.out) == b.stored_len
        return
    assert b.tokens and b.tokens[-1] == EOB and EOB not in b.tokens[:-1]
    for t in b.tokens:
        if isinstance(t, tuple):
            assert 3 <= t[0] <= 258 and 1 <= t[1] <= 32768
    if b.btype == 2:
        assert 257 <= b.hlit <= 286 and 1 <= b.hdist <= 30 and 4 <= b.hclen <= 19
        assert len(b.ll_lens) == b.hlit and len(b.d_lens) == b.hdist and len(b.cl_lens) == 19
        assert all(b.cl_lens[CL_ORDER[i]] == 0 for i in range(b.hclen, 19))
        lens = []
        for y, x in b.rle:                     # the header's run-length symbols expand to the two length vectors
            lens += [y] if y < 16 else [lens[-1]] * (3 + x) if y == 16 else [0] * ((3 if y == 17 else 11) + x)
        assert lens == b.ll_lens + b.d_lens


@pytest.mark.parametrize('kind,v', SETTINGS)
@pytest.mark.parametrize('name', sorted(CORPUS))
def test_inflate_blocks_matches_zlib(name, kind, v):
    data = CORPUS[name]
    z = _compress(data, kind, v)
    blocks = inflate_blocks(z)
    assert b''.join(b.out for b in blocks) == zlib.decompress(z) == data
    assert [b.final for b in blocks] == [False] * (len(blocks) - 1) + [True]
    pos, start = 0, 0
    for b in blocks:
        _check_block(b)
        assert b.start_bit == start and b.end_bit > b.start_bit and b.out_start == pos
        if b.tokens:                            # the tokens replay to the block's bytes, with the stream so far as window
            assert replay(b.tokens, data[:pos]) == b.out
        pos += len(b.out)
        start = b.end_bit
    assert 8 * (len(z) - 6) - 7 <= blocks[-1].end_bit <= 8 * (len(z) - 6)


def test_inflate_covers_every_block_type():
    seen = set()
    for name in CORPUS:
        for kind, v in SETTINGS:
            seen |= {b.btype for b in inflate_blocks(_compress(CORPUS[name], kind, v))}
    assert seen == {0, 1, 2}
    blocks = inflate_blocks(zlib.compress(CORPUS['far'], 9))
    assert any(isinstance(t, tuple) and t[1] > 30000 for b in blocks for t in b.tokens)


def test_flush_blocks_and_sync_markers():
    """Z_SYNC_FLUSH ends with an empty stored block, byte-aligned and not final; the stream goes on after it."""
    c = zlib.compressobj(6)
    z = c.compress(CORPUS['text'][:50000]) + c.flush(zlib.Z_SYNC_FLUSH) + c.compress(CORPUS['skew']) + c.flush()
    blocks = inflate_blocks(z)
    empty = [b for b in blocks if b.btype == 0 and b.stored_len == 0]
    assert empty and not empty[0].final and empty[0].end_bit % 8 == 0
    assert b''.join(b.out for b in blocks) == CORPUS['text'][:50000] + CORPUS['skew']


def test_histograms_and_codes():
    toks = [65, 66, (3, 1), (258, 2), (10, 32768), (4, 5), EOB]
    ll, d = histograms(toks)
    assert ll[65] == ll[66] == 1 and ll[EOB] == 1 and sum(ll) == 7
    assert ll[257] == 1 and ll[285] == 1 and ll[257 + 7] == 1 and ll[258] == 1
    assert d[0] == 1 and d[1] == 1 and d[29] == 1 and d[4] == 1 and sum(d) == 4
    # RFC 1951 3.2.5's table, at the edges of every code
    assert [len_code(x) for x in (3, 10, 11, 12, 13, 18, 19, 34, 35, 66, 67, 130, 131, 226, 227, 257, 258)] == \
        [0, 7, 8, 8, 9, 11, 12, 15, 16, 19, 20, 23, 24, 26, 27, 27, 28]
    assert [dist_code(x) for x in (1, 4, 5, 6, 7, 8, 9, 12, 13, 24, 25, 4096, 4097, 24576, 24577, 32768)] == \
        [0, 3, 4, 4, 5, 5, 6, 6, 7, 8, 9, 23, 24, 28, 29, 29]
    assert at_least_two([0] * 30)[:2] == [1, 1]
    assert at_least_two([0, 0, 5])[:3] == [1, 0, 5]
    assert at_least_two([5, 0, 0])[:3] == [5, 1, 0]
    assert at_least_two([0, 5, 0]) == [1, 5, 0]
    assert at_least_two([2, 3, 0]) == [2, 3, 0]


# ---- corrupted streams ---------------------------------------------------------------------------------------

def _dynamic_stream():
    z = zlib.compress(CORPUS['skew'][:20000], 9)
    assert inflate_blocks(z)[0].btype == 2
    return z


def _flip(z, bit):
    b = bytearray(z)
    b[bit >> 3] ^= 1 << (bit & 7)
    return bytes(b)


@pytest.mark.parametrize('bit', range(16, 16 + 3 + 14))
def test_rejects_a_flipped_header_bit(bit):
    """A flipped bit of BTYPE / HLIT / HDIST / HCLEN of a dynamic block: the stream no longer decodes to the input, and
    the decoder says so (reserved type, inconsistent code, overrun, wrong Adler-32 or trailing bytes)."""
    z = _dynamic_stream()
    with pytest.raises(InflateError):
        inflate_blocks(_flip(z, bit))


def test_rejects_flipped_zlib_header_and_adler():
    z = _dynamic_stream()
    for bit in (0, 3, 8 + 5):                   # CM, FDICT / FCHECK
        with pytest.raises(InflateError):
            inflate_blocks(_flip(z, bit))
    with pytest.raises(InflateError, match='Adler'):
        inflate_blocks(_flip(z, 8 * len(z) - 1))


def _bits_to_bytes(bits):
    out = bytearray((len(bits) + 7) // 8)
    for i, v in enumerate(bits):
        out[i >> 3] |= v << (i & 7)
    return bytes(out)


def _put(bits, v, n):
    bits += [(v >> k) & 1 for k in range(n)]


def _dynamic_block(cl_lens, ll_lens, d_lens):
    """A final dynamic block's header with the given lengths, every code length sent as a literal 0..15 symbol; the
    code-length code's canonical codes come from cl_lens (which must give every length used a code)."""
    bits = [1, 0, 1]
    _put(bits, len(ll_lens) - 257, 5)
    _put(bits, len(d_lens) - 1, 5)
    _put(bits, 15, 4)
    for i in range(19):
        _put(bits, cl_lens[CL_ORDER[i]], 3)
    cnt = [0] * 8
    for l in cl_lens:
        cnt[l] += 1
    cnt[0] = 0
    nxt, c = [0] * 8, 0
    for l in range(1, 8):
        c = (c + cnt[l - 1]) << 1
        nxt[l] = c
    code = {}
    for s, l in enumerate(cl_lens):
        if l:
            code[s] = (nxt[l], l)
            nxt[l] += 1
    for v in list(ll_lens) + list(d_lens):
        cv, l = code[v]
        bits += [(cv >> (l - 1 - k)) & 1 for k in range(l)]       # Huffman codes go MSB first
    return bits


def test_rejects_oversubscribed_and_incomplete_codes():
    cl = [0] * 19
    cl[1] = cl[2] = cl[0] = 2; cl[3] = 2           # four 2-bit codes: complete
    ok_ll = [0] * 257
    ok_ll[65], ok_ll[EOB] = 1, 1
    hdr = _dynamic_block(cl, ok_ll, [1, 1])
    # the header decodes; the first data bit then selects 'A' (code 0) or EOB (code 1)
    z = b'\x78\x9c' + _bits_to_bytes(hdr + [1])
    with pytest.raises(InflateError, match='Adler|truncated'):
        inflate_blocks(z)
    z = b'\x78\x9c' + _bits_to_bytes(hdr + [1]) + zlib.adler32(b'').to_bytes(4, 'big')
    assert inflate_blocks(z)[0].out == b''
    over_ll = list(ok_ll)
    over_ll[66] = 1                                # three 1-bit codes
    with pytest.raises(InflateError, match='over-subscribed'):
        inflate_blocks(b'\x78\x9c' + _bits_to_bytes(_dynamic_block(cl, over_ll, [1, 1]) + [0] * 40))
    inc_ll = list(ok_ll)
    inc_ll[65] = 2                                 # 1 + 2 bits: a quarter of the code space unused
    with pytest.raises(InflateError, match='incomplete'):
        inflate_blocks(b'\x78\x9c' + _bits_to_bytes(_dynamic_block(cl, inc_ll, [1, 1]) + [0] * 40))
    with pytest.raises(InflateError, match='over-subscribed'):
        inflate_blocks(b'\x78\x9c' + _bits_to_bytes(_dynamic_block(cl, ok_ll, [1, 1, 1]) + [0] * 40))
    with pytest.raises(InflateError, match='incomplete'):
        inflate_blocks(b'\x78\x9c' + _bits_to_bytes(_dynamic_block(cl, ok_ll, [2, 1, 0]) + [0] * 40))
    # one distance code of one bit (RFC 1951 3.2.7) is allowed, so is none at all
    for d in ([1], [0, 1], [0]):
        z = b'\x78\x9c' + _bits_to_bytes(_dynamic_block(cl, ok_ll, d) + [1]) + zlib.adler32(b'').to_bytes(4, 'big')
        assert inflate_blocks(z)[0].d_lens == d
    bad_cl = list(cl)
    bad_cl[4] = 2                                  # five 2-bit codes: the code-length code itself over-subscribed
    with pytest.raises(InflateError, match='over-subscribed'):
        inflate_blocks(b'\x78\x9c' + _bits_to_bytes(_dynamic_block(bad_cl, ok_ll, [1, 1]) + [0] * 40))


def test_rejects_far_distance_bad_stored_and_truncation():
    # fixed block: literal 'a' then a match of length 3 at distance 2 (one byte out so far)
    bits = [1, 1, 0]
    lit = 0x30 + ord('a')                          # 8-bit codes 00110000 + literal
    bits += [(lit >> (7 - k)) & 1 for k in range(8)]
    bits += [0, 0, 0, 0, 0, 0, 1]                  # 7-bit code of symbol 257 (length 3)
    bits += [0, 0, 0, 0, 1]                        # 5-bit distance code 1 (distance 2)
    bits += [0] * 7                                # EOB
    with pytest.raises(InflateError, match='before the stream start'):
        inflate_blocks(b'\x78\x9c' + _bits_to_bytes(bits) + b'\0' * 4)
    z = zlib.compress(b'stored bytes', 0)
    assert inflate_blocks(z)[0].btype == 0
    b = bytearray(z)
    b[5] ^= 1                                      # NLEN's low byte
    with pytest.raises(InflateError, match='LEN'):
        inflate_blocks(bytes(b))
    for k in (3, 7, len(z) - 5, len(z) - 1):
        with pytest.raises(InflateError):
            inflate_blocks(z[:k])
    zd = _dynamic_stream()
    for k in (4, 40, len(zd) // 2, len(zd) - 5, len(zd) - 1):
        with pytest.raises(InflateError):
            inflate_blocks(zd[:k])
    with pytest.raises(InflateError, match='after the stream'):
        inflate_blocks(zd + b'\0')


# ---- optimal_limited_cost ----------------------------------------------------------------------------------

def _exhaustive(freq, maxbits):
    f = np.array([x for x in freq if x > 0], np.int64)
    m = len(f)
    if m <= 1:
        return int(f.sum())
    L = np.array(list(itertools.product(range(1, maxbits + 1), repeat=m)), np.int64)
    kraft = (np.int64(1) << (maxbits - L)).sum(1) <= (1 << maxbits)
    if not kraft.any():
        return None
    return int((L[kraft] * f).sum(1).min())


def _fib(m):
    a, b, out = 1, 1, []
    for _ in range(m):
        out.append(a)
        a, b = b, a + b
    return out


def _cases():
    g = np.random.default_rng(3)
    cases = []
    for m in range(1, 8):
        cases.append(_fib(m))
        for _ in range(3):
            cases.append(g.integers(1, 50, m).tolist())
        cases.append(g.integers(1, 1000, m).tolist())
        cases.append([1] * m)
    cases.append([0, 3, 0, 0, 1, 9, 0])                 # zeros between the symbols
    cases.append([2 ** k for k in range(7)])
    return cases


@pytest.mark.parametrize('maxbits', [2, 3, 4, 5])
def test_optimal_limited_cost_equals_exhaustive_search(maxbits):
    tried = binding = 0
    for freq in _cases():
        want = _exhaustive(freq, maxbits)
        if want is None:                                 # more symbols than 2^maxbits codes
            with pytest.raises(ValueError):
                optimal_limited_cost(freq, maxbits)
            continue
        got = optimal_limited_cost(freq, maxbits)
        assert got == want, (freq, maxbits)
        assert got >= huffman_cost(freq)
        tried += 1
        binding += got > huffman_cost(freq)
    assert tried >= 20 and binding >= (3 if maxbits <= 4 else 0)


def test_huffman_cost_is_the_unlimited_optimum():
    for freq in _cases():
        nz = sum(f > 0 for f in freq)
        if nz <= 6:                                      # an optimal code is at most m - 1 deep
            assert huffman_cost(freq) == _exhaustive(freq, max(1, nz - 1))
        assert optimal_limited_cost(freq, 15) == huffman_cost(freq)
    # Fibonacci weights: the Huffman tree is a chain of depth m - 1, so a limit below m - 1 costs bits
    f = _fib(20)
    assert optimal_limited_cost(f, 19) == huffman_cost(f) < optimal_limited_cost(f, 18) < optimal_limited_cost(f, 15)
    assert optimal_limited_cost([5, 5, 5, 5], 2) == 40 and optimal_limited_cost([7], 3) == 7
    assert optimal_limited_cost([0, 0], 3) == 0
