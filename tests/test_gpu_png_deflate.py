"""GPU: the deflate stage of the PNG encoder (csrc/k4_png.cu) checked below its output.

(a) k4_testing_png_code_lengths runs the encoder's own package-merge on histograms no frame produces -- Fibonacci counts
whose Huffman code is deeper than the 15- or 7-bit limit, geometric, Zipf, flat, two-symbol, tied and sparse ones -- and
the lengths are checked against the optimal length-limited cost (tests/deflate_ref.py's package-merge, pinned against
an exhaustive search by tests/test_deflate_ref.py).

(b) Whole files from png_encode, their IDAT parsed block by block by deflate_ref.inflate_blocks: one block per
K4_PNG_SEG segment holding exactly that segment's filtered bytes, the empty stored block after every dynamic segment but
the last, BFINAL on the last block only; every dynamic block's three codes optimal for the histograms recounted from its
own tokens and header, HLIT / HDIST / HCLEN minimal, the dynamic block chosen only when smaller than the stored one, and
the match finder's length and distance rules.  Which frames make a length limit bind is printed per file (pytest -s).
"""
import ctypes as C
import struct

import numpy as np
import pytest
import torch

import k4nerf
from k4nerf import _lib, render
from k4nerf.utils import png_encode
from deflate_ref import (CL_ORDER, at_least_two, code_cost, histograms, huffman_cost, inflate_blocks,
                         optimal_limited_cost)
from helpers import make_state, model_from_state
from oracle import scenes, sftnet
from png_ref import filter_np

pytestmark = pytest.mark.gpu
SEG = _lib.K4_PNG_SEG


# ---- (a) code lengths of chosen histograms ---------------------------------------------------------------

def _code_lengths(freq, maxbits, dev):
    f = torch.tensor(freq, dtype=torch.int32, device=dev)
    out = torch.full((len(freq),), 0xee, dtype=torch.uint8, device=dev)
    _lib.check(_lib.lib.k4_testing_png_code_lengths(C.c_void_p(f.data_ptr()), len(freq), maxbits,
                                                     C.c_void_p(out.data_ptr()),
                                                     C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    return out.cpu().tolist()


def _check_code(freq, lens, maxbits, what):
    """lens is an optimal complete prefix code of the non-zero counts of freq with no length above maxbits."""
    f = np.asarray(freq, np.int64)
    ln = np.asarray(lens, np.int64)
    assert ln.max() <= maxbits, (what, 'length above the limit', int(ln.max()))
    assert np.array_equal(f > 0, ln > 0), (what, 'a code for a zero count or none for a non-zero one')
    assert int((np.int64(1) << (15 - ln[ln > 0])).sum()) == 1 << 15, (what, 'Kraft sum is not 1')
    nz = np.flatnonzero(f > 0)
    fi, li = f[nz], ln[nz]
    assert not ((fi[:, None] > fi[None, :]) & (li[:, None] > li[None, :])).any(), (what, 'larger count, longer code')
    assert code_cost(freq, lens) == optimal_limited_cost(freq, maxbits), (what, 'cost above the optimum')


def _fib(m):
    a, b, out = 1, 1, []
    for _ in range(m):
        out.append(a)
        a, b = b, a + b
    return out


def _place(counts, n, seed):
    """counts at n slots chosen by a seeded permutation, zeros elsewhere."""
    f = [0] * n
    for slot, c in zip(np.random.default_rng(seed).permutation(n)[:len(counts)], counts):
        f[int(slot)] = int(c)
    return f


def _fib_cases():
    for m in range(17, 22):
        yield f'fib{m}/n286', _place(_fib(m), 286, m), 15
        yield f'fib{m}/n30', _place(_fib(m), 30, m), 15
    for m in range(9, 20):
        yield f'fib{m}/n19', _place(_fib(m), 19, m), 7


@pytest.mark.parametrize('name,freq,maxbits', list(_fib_cases()), ids=lambda v: v if isinstance(v, str) else '')
def test_code_lengths_where_the_limit_binds(cuda_device, name, freq, maxbits):
    """Fibonacci counts over m symbols: the Huffman code is a chain m - 1 deep, beyond the limit, so the limit binds."""
    assert sum(freq) <= SEG + 1 or maxbits == 7            # a segment's tokens plus EOB could give these counts
    lens = _code_lengths(freq, maxbits, cuda_device)
    _check_code(freq, lens, maxbits, name)
    assert huffman_cost(freq) < code_cost(freq, lens), name
    assert max(lens) == maxbits, name


def _shaped_cases():
    g = np.random.default_rng(11)
    k = np.arange(286)
    yield 'geometric', np.round(20000 * 0.8 ** k).astype(int).tolist(), 15
    yield 'geometric/n30', np.round(9000 * 0.6 ** k[:30]).astype(int).tolist(), 15
    yield 'zipf', np.round(30000 / (k + 1)).astype(int).tolist(), 15
    yield 'zipf/n19', np.round(5000 / (k[:19] + 1) ** 1.5).astype(int).tolist(), 7
    yield 'flat286', [100] * 286, 15
    yield 'flat19', [7] * 19, 7
    yield 'flat30', [1] * 30, 15
    yield 'two', _place([5, 1], 286, 1), 15
    yield 'two/first', [1, 1] + [0] * 28, 15
    yield 'two/last', [0] * 17 + [300, 2], 7
    yield 'ties', (g.integers(1, 4, 286) * 1000).tolist(), 15
    yield 'ties/n19', [5, 5, 5, 5, 1, 1, 1, 1, 9, 9, 0, 0, 2, 2, 2, 2, 2, 2, 2], 7
    yield 'sparse', [int(x) * (i % 3 == 0) for i, x in enumerate(g.integers(1, 2000, 286))], 15
    yield 'sparse/n30', [0, 9, 0, 0, 4, 0, 0, 0, 1, 0, 0, 0, 0, 70, 0, 0, 0, 0, 0, 3, 0, 0, 2, 0, 0, 0, 0, 0, 0, 1], 15
    yield 'random/n19/limit6', g.integers(1, 30000, 19).tolist(), 6
    yield 'skewed/n19/limit5', [2 ** min(i, 14) for i in range(16)] + [0, 0, 0], 5
    yield 'negative', [-5, 3, 0, 2, -1, 1] + [0] * 24, 15


@pytest.mark.parametrize('name,freq,maxbits', list(_shaped_cases()), ids=lambda v: v if isinstance(v, str) else '')
def test_code_lengths_are_optimal(cuda_device, name, freq, maxbits):
    lens = _code_lengths(freq, maxbits, cuda_device)
    pos = [max(0, x) for x in freq]
    _check_code(pos, lens, maxbits, name)


def test_code_lengths_refuse_what_package_merge_cannot_code(cuda_device):
    """More non-zero counts than 2^maxbits codes, or a total count too large for the 32-bit item weights: 0xff."""
    assert _code_lengths([1] * 20 + [0] * 10, 4, cuda_device) == [0xff] * 30
    assert _code_lengths([2 ** 30, 2 ** 30, 5], 15, cuda_device) == [0xff] * 3
    lens = _code_lengths([1] * 8 + [0] * 11, 4, cuda_device)    # eight codes fit in four bits
    _check_code([1] * 8 + [0] * 11, lens, 4, 'eight')


# ---- (b) whole files --------------------------------------------------------------------------------------

def _idat(data):
    pos, idat = 8, b''
    while pos < len(data):
        n, = struct.unpack('>I', data[pos:pos + 4])
        if data[pos + 4:pos + 8] == b'IDAT':
            idat += data[pos + 8:pos + 8 + n]
        pos += 12 + n
    return idat


def _binds(freq, lens):
    return code_cost(freq, lens) > huffman_cost(freq)


def _check_file(frame, dev, name):
    """Encode frame on the device and check its deflate stream block by block; return the tally of the file."""
    frame = np.ascontiguousarray(frame)
    data = png_encode(torch.from_numpy(frame).to(dev))
    filt = filter_np(frame).tobytes()
    n = len(filt)
    nseg = -(-n // SEG)
    blocks = inflate_blocks(_idat(data))
    tally = dict(stored=0, dynamic=0, ll15=0, d15=0, cl7=0, far=0)
    i = 0
    for k in range(nseg):
        lo, hi = k * SEG, min(n, (k + 1) * SEG)
        b = blocks[i]
        i += 1
        where = f'{name}: segment {k}'
        # layout: one stored or dynamic block per segment, byte-aligned, holding exactly the segment's bytes
        assert b.btype in (0, 2), where
        assert b.start_bit % 8 == 0 and b.out_start == lo and b.out == filt[lo:hi], where
        assert b.final == (k == nseg - 1), where
        end = b.end_bit
        if b.btype == 2 and k < nseg - 1:
            sync = blocks[i]
            i += 1
            assert sync.btype == 0 and sync.stored_len == 0 and not sync.final, where
            end = sync.end_bit
        size = (end - b.start_bit + 7) // 8
        if b.btype == 0:
            tally['stored'] += 1
            assert size == 5 + hi - lo, where
            continue
        tally['dynamic'] += 1
        # choice: the dynamic block and its sync block are smaller than the stored block
        assert size < 5 + hi - lo, (where, size)
        # codes: optimal for the block's own tokens and header
        ll, d = histograms(b.tokens)
        assert ll[256] == 1, where
        d = at_least_two(d)
        ll_lens = b.ll_lens + [0] * (286 - b.hlit)
        d_lens = b.d_lens + [0] * (30 - b.hdist)
        _check_code(ll, ll_lens, 15, where + ' literal / length code')
        _check_code(d, d_lens, 15, where + ' distance code')
        cl = [0] * 19
        for y, _ in b.rle:
            cl[y] += 1
        cl = at_least_two(cl)
        _check_code(cl, b.cl_lens, 7, where + ' code-length code')
        assert b.hlit == 257 or b.ll_lens[-1], (where, 'HLIT not minimal', b.hlit)
        assert b.hdist == 1 or b.d_lens[-1], (where, 'HDIST not minimal', b.hdist)
        assert b.hclen == 4 or b.cl_lens[CL_ORDER[b.hclen - 1]], (where, 'HCLEN not minimal', b.hclen)
        tally['ll15'] += _binds(ll, ll_lens)
        tally['d15'] += _binds(d, d_lens)
        tally['cl7'] += _binds(cl, b.cl_lens)
        # matches: length 3..258, distance 1..32768, no length-3 match beyond 4096
        p = lo
        for t in b.tokens:
            if isinstance(t, tuple):
                ln, dist = t
                assert 3 <= ln <= 258 and 1 <= dist <= 32768 and not (ln == 3 and dist > 4096), (where, p, t)
                tally['far'] += p - dist < lo
                p += ln
            else:
                p += t != 256
        assert p == hi, where
    assert i == len(blocks), name
    print(f'\n{name}: {n} bytes, {nseg} segments, stored {tally["stored"]} dynamic {tally["dynamic"]}; limit binding in '
          f'literal/length (15) {tally["ll15"]}, distance (15) {tally["d15"]}, code-length (7) {tally["cl7"]} blocks; '
          f'{tally["far"]} matches into the previous segment')
    return tally


def _rng(seed):
    return np.random.default_rng(seed)


def _smooth(H, W, seed):
    """test_gpu_png.py's shapes frame: a smooth pattern with noise in -2..2."""
    g = _rng(seed)
    yy, xx = np.mgrid[0:H, 0:W]
    s = np.stack([(xx * 3 + yy) % 256, (xx + 2 * yy) % 256, (xx * yy) % 256], -1)
    return np.clip(s + g.integers(-2, 3, s.shape), 0, 255).astype(np.uint8)


@pytest.mark.parametrize('H,W', [(1, 1), (1, 7), (1, 1000), (9, 1), (700, 1), (5, 5), (37, 41), (63, 129), (100, 333)])
def test_blocks_of_shapes(cuda_device, H, W):
    _check_file(_smooth(H, W, H * 1000 + W), cuda_device, f'shape {H}x{W}')


@pytest.mark.parametrize('H,W,nbytes', [(1, 21845, 2 * SEG), (24576, 1, 3 * SEG), (1, 32768, 3 * SEG + 1),
                                         (1, 43690, 4 * SEG - 1), (2, 5461, SEG)])
def test_blocks_at_segment_boundaries(cuda_device, H, W, nbytes):
    assert H * (1 + 3 * W) == nbytes
    f = (np.arange(H * W * 3).reshape(H, W, 3) // 7 % 256).astype(np.uint8)
    f[..., 1] ^= _rng(W).integers(0, 4, (H, W), dtype=np.uint8)
    _check_file(f, cuda_device, f'boundary {H}x{W}')


@pytest.mark.parametrize('value', [0, 1, 200])
@pytest.mark.parametrize('H,W', [(1, 70000), (300, 301), (32, 4032)])
def test_constant_frames_take_dynamic_blocks(cuda_device, value, H, W):
    t = _check_file(np.full((H, W, 3), value, np.uint8), cuda_device, f'constant {value} {H}x{W}')
    assert t['stored'] == 0


def test_matches_at_distance_32768_reach_the_previous_segment(cuda_device):
    """Rows A, B, A, B, ... of random bytes with 1 + 3 W = 16384: from row 2 on the filtered stream repeats with a period
    of exactly one segment, so segments 2.. are dynamic and code their bytes as matches into the segment before."""
    g = _rng(5)
    W = 5461
    a, b = g.integers(0, 256, (2, W, 3), dtype=np.uint8)
    t = _check_file(np.stack([a if y % 2 == 0 else b for y in range(24)]), cuda_device, 'distance 32768')
    assert t['dynamic'] >= 10 and t['far'] >= 10


@pytest.mark.parametrize('H,W', [(1, 1), (17, 19), (128, 1000)])
def test_uniform_noise_takes_only_stored_blocks(cuda_device, H, W):
    t = _check_file(_rng(H + W).integers(0, 256, (H, W, 3), dtype=np.uint8), cuda_device, f'noise {H}x{W}')
    assert t['dynamic'] == 0


def test_smooth_gradient_takes_only_dynamic_blocks(cuda_device):
    H, W = 128, 1000
    yy, xx = np.mgrid[0:H, 0:W]
    s = np.stack([xx // 4 + yy // 3, xx // 5 + 2 * yy, xx // 7 + yy], -1) % 256
    f = np.clip(s + _rng(8).integers(-2, 3, s.shape), 0, 255).astype(np.uint8)
    t = _check_file(f, cuda_device, f'gradient {H}x{W}')
    assert t['stored'] == 0


def test_decoder_frame_band(cuda_device):
    """Rows 1024..1279 of test_gpu_png.py's seeded 4032 x 3024 decoder frame."""
    m = model_from_state(make_state('cfgA', res=48, regime='shell'), cuda_device)
    net = k4nerf.SFTNet(3, 4, 64, 5, 32, 1)
    net.load_state_dict(sftnet.random_state_dict(seed=3))
    net = net.to(cuda_device)
    K, c2w = scenes.blender_camera(756, 1008, theta=40.0)
    u8, _ = render.render_frame_4k(m, net, 756, 1008, K, c2w.numpy(), False, dict(scenes.RENDER_KW_DVGO), out_u8=True)
    assert tuple(u8.shape) == (3024, 4032, 3)
    _check_file(u8[1024:1280].cpu().numpy(), cuda_device, 'decoder frame rows 1024..1279')
