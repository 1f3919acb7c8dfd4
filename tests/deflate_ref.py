"""Plain-Python references for the tests of the deflate stage of csrc/k4_png.cu.

inflate_blocks: an instrumented zlib (RFC 1950) / deflate (RFC 1951) decoder that returns every block as it was coded --
its type, BFINAL, bit extent, for a dynamic block the whole header (HLIT / HDIST / HCLEN, the code-length code, the
run-length symbols and the two code-length vectors), the decoded tokens and the block's output bytes.  It is strict: an
over-subscribed code, an incomplete one (outside RFC 1951's one-distance-code case), a distance reaching before the
stream's start, a bad stored LEN / NLEN, a reserved block type, an invalid symbol, a wrong Adler-32, a truncated stream
or bytes after it raise InflateError.

optimal_limited_cost: the least sum f_i l_i over prefix codes of the non-zero frequencies with every l_i <= maxbits,
from Larmore and Hirschberg's package-merge ("A fast algorithm for optimal length-limited Huffman codes", JACM 1990):
the cost is the total weight of the 2 m - 2 lightest items of the last merged list.  huffman_cost: the same without
the limit, by Huffman's algorithm.  Costs, not length vectors, are compared: several optimal length vectors can exist,
the cost is unique.
"""
import heapq
import zlib
from dataclasses import dataclass, field

# RFC 1951 3.2.5: base value and extra bits of the length codes 257..285 and the distance codes 0..29
LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227,
            258]
LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
             6145, 8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0] + [k // 2 for k in range(2, 28)]
# RFC 1951 3.2.7: the order of the code-length code's lengths in a dynamic block's header
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
EOB = 256

_LEN_CODE = [0] * 259                  # length 3..258 -> 0..28 (the code 257 + i)
for _i in range(29):
    for _l in range(LEN_BASE[_i], LEN_BASE[_i] + (1 << LEN_EXTRA[_i])):
        if _l <= 258:
            _LEN_CODE[_l] = _i
_LEN_CODE[258] = 28                    # 258 has its own code; 227 + 31 under code 27 is not used
_DIST_CODE = [0] * 32769               # distance 1..32768 -> 0..29
for _i in range(30):
    for _d in range(DIST_BASE[_i], DIST_BASE[_i] + (1 << DIST_EXTRA[_i])):
        _DIST_CODE[_d] = _i


def len_code(length):
    """The length code (0..28; the literal / length symbol is 257 + it) of a match length 3..258."""
    return _LEN_CODE[length]


def dist_code(dist):
    """The distance code (0..29) of a distance 1..32768."""
    return _DIST_CODE[dist]


class InflateError(ValueError):
    pass


@dataclass
class Block:
    """One deflate block.  ``btype`` 0 stored, 1 fixed, 2 dynamic; ``start_bit`` / ``end_bit`` are offsets into the
    deflate data (after the zlib header), the end after the EOB code or the stored bytes.  ``tokens``: literals as ints
    0..255, matches as (length, distance) tuples, and EOB (256) last; a stored block has none.  ``out_start``: the
    offset of the block's first output byte in the whole stream.  Dynamic blocks only: ``hlit``, ``hdist``, ``hclen``
    as counts (257.., 1.., 4..), ``cl_lens`` the code-length code's 19 lengths by symbol, ``rle`` its symbols as (symbol,
    extra value) pairs in header order, ``ll_lens`` / ``d_lens`` the HLIT and HDIST code lengths.  ``stored_len``: LEN of
    a stored block."""
    btype: int
    final: bool
    start_bit: int
    end_bit: int = 0
    out_start: int = 0
    out: bytes = b''
    tokens: list = field(default_factory=list)
    stored_len: int = 0
    hlit: int = 0
    hdist: int = 0
    hclen: int = 0
    cl_lens: list = field(default_factory=list)
    rle: list = field(default_factory=list)
    ll_lens: list = field(default_factory=list)
    d_lens: list = field(default_factory=list)


def _decode_table(lens, kind, allow_single=False):
    """(table, maxlen) for LSB-first canonical decoding: table[next maxlen bits] = (symbol, length) or None.  Raises on
    an over-subscribed code and on an incomplete one, except (allow_single) one code of length 1 or no code at all."""
    maxlen = max(lens) if lens else 0
    if maxlen == 0:
        if allow_single:
            return [None], 0
        raise InflateError(f'{kind}: no codes')
    if maxlen > 15:
        raise InflateError(f'{kind}: length {maxlen} > 15')
    count = [0] * 16
    for l in lens:
        count[l] += 1
    left = 1
    for l in range(1, 16):
        left = 2 * left - count[l]
        if left < 0:
            raise InflateError(f'{kind}: over-subscribed code')
    if left > 0 and not (allow_single and maxlen == 1 and count[1] == 1):
        raise InflateError(f'{kind}: incomplete code')
    nxt, c = [0] * 16, 0
    for l in range(1, 16):
        c = (c + count[l - 1]) << 1 if l > 1 else 0
        nxt[l] = c
    table = [None] * (1 << maxlen)
    for sym, l in enumerate(lens):
        if l:
            code = nxt[l]
            nxt[l] += 1
            r = int(format(code, f'0{l}b')[::-1], 2)
            table[r::1 << l] = [(sym, l)] * (1 << (maxlen - l))
    return table, maxlen


_FIXED = None


def _fixed_tables():
    global _FIXED
    if _FIXED is None:
        ll = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
        _FIXED = (_decode_table(ll, 'fixed literal / length'), _decode_table([5] * 32, 'fixed distance'))
    return _FIXED


class _Bits:
    def __init__(self, data, pos):
        self.data = bytes(data) + b'\0' * 8
        self.nbits = 8 * len(data)
        self.pos = pos

    def need(self):
        if self.pos > self.nbits:
            raise InflateError('truncated stream')

    def get(self, n):
        p = self.pos
        v = (int.from_bytes(self.data[p >> 3:(p >> 3) + 4], 'little') >> (p & 7)) & ((1 << n) - 1)
        self.pos = p + n
        self.need()
        return v

    def sym(self, table, maxlen, kind):
        p = self.pos
        e = table[(int.from_bytes(self.data[p >> 3:(p >> 3) + 4], 'little') >> (p & 7)) & ((1 << maxlen) - 1)]
        if e is None:
            raise InflateError(f'{kind}: unused code')
        self.pos = p + e[1]
        self.need()
        return e[0]


def _dynamic_header(bits, blk):
    blk.hlit = bits.get(5) + 257
    blk.hdist = bits.get(5) + 1
    blk.hclen = bits.get(4) + 4
    if blk.hlit > 286 or blk.hdist > 30:
        raise InflateError(f'HLIT {blk.hlit} / HDIST {blk.hdist} out of range')
    cl = [0] * 19
    for i in range(blk.hclen):
        cl[CL_ORDER[i]] = bits.get(3)
    blk.cl_lens = cl
    table, ml = _decode_table(cl, 'code-length code')
    n = blk.hlit + blk.hdist
    lens = []
    while len(lens) < n:
        y = bits.sym(table, ml, 'code-length code')
        if y < 16:
            blk.rle.append((y, 0))
            lens.append(y)
            continue
        if y == 16:
            if not lens:
                raise InflateError('repeat with no previous length')
            x = bits.get(2)
            v, r = lens[-1], 3 + x
        elif y == 17:
            x = bits.get(3)
            v, r = 0, 3 + x
        else:
            x = bits.get(7)
            v, r = 0, 11 + x
        blk.rle.append((y, x))
        if len(lens) + r > n:
            raise InflateError('code lengths overrun HLIT + HDIST')
        lens += [v] * r
    blk.ll_lens, blk.d_lens = lens[:blk.hlit], lens[blk.hlit:]
    if blk.ll_lens[EOB] == 0:
        raise InflateError('no end-of-block code')
    return _decode_table(blk.ll_lens, 'literal / length'), _decode_table(blk.d_lens, 'distance', allow_single=True)


def _codes(bits, blk, out, lt, dt):
    (ltab, lml), (dtab, dml) = lt, dt
    toks = blk.tokens
    data, nbits = bits.data, bits.nbits
    p = bits.pos
    while True:
        e = ltab[(int.from_bytes(data[p >> 3:(p >> 3) + 4], 'little') >> (p & 7)) & ((1 << lml) - 1)]
        if e is None:
            raise InflateError('literal / length: unused code')
        y, p = e[0], p + e[1]
        if y < 256:
            out.append(y)
            toks.append(y)
        elif y == EOB:
            toks.append(EOB)
            break
        else:
            y -= 257
            if y >= 29:
                raise InflateError(f'invalid length symbol {y + 257}')
            w = int.from_bytes(data[p >> 3:(p >> 3) + 8], 'little') >> (p & 7)
            ne = LEN_EXTRA[y]
            length = LEN_BASE[y] + (w & ((1 << ne) - 1))
            p += ne
            e = dtab[(int.from_bytes(data[p >> 3:(p >> 3) + 4], 'little') >> (p & 7)) & ((1 << dml) - 1)]
            if e is None:
                raise InflateError('distance: unused code')
            dc, p = e[0], p + e[1]
            if dc >= 30:
                raise InflateError(f'invalid distance symbol {dc}')
            ne = DIST_EXTRA[dc]
            dist = DIST_BASE[dc] + ((int.from_bytes(data[p >> 3:(p >> 3) + 4], 'little') >> (p & 7)) & ((1 << ne) - 1))
            p += ne
            if dist > len(out):
                raise InflateError(f'distance {dist} before the stream start ({len(out)} bytes out)')
            s = len(out) - dist
            if dist >= length:
                out += out[s:s + length]
            else:
                for k in range(length):
                    out.append(out[s + k])
            toks.append((length, dist))
        if p > nbits:
            raise InflateError('truncated stream')
    bits.pos = p
    bits.need()


def inflate_blocks(zdata):
    """The blocks of a zlib stream (list of Block), after checking its header, its Adler-32 and that nothing follows."""
    zdata = bytes(zdata)
    if len(zdata) < 6:
        raise InflateError('truncated stream')
    cmf, flg = zdata[0], zdata[1]
    if cmf & 15 != 8 or cmf >> 4 > 7 or (cmf * 256 + flg) % 31 or flg & 32:
        raise InflateError('bad zlib header')
    body = zdata[2:]
    bits = _Bits(body, 0)
    out = bytearray()
    blocks = []
    final = False
    while not final:
        blk = Block(btype=-1, final=False, start_bit=bits.pos, out_start=len(out))
        final = blk.final = bool(bits.get(1))
        blk.btype = bits.get(2)
        if blk.btype == 0:
            bits.pos = (bits.pos + 7) & ~7
            ln, nln = bits.get(16), bits.get(16)
            if ln != nln ^ 0xffff:
                raise InflateError(f'stored LEN {ln:#06x} / NLEN {nln:#06x}')
            a = bits.pos >> 3
            bits.pos += 8 * ln
            bits.need()
            blk.stored_len = ln
            out += body[a:a + ln]
        elif blk.btype == 1:
            _codes(bits, blk, out, *_fixed_tables())
        elif blk.btype == 2:
            lt, dt = _dynamic_header(bits, blk)
            _codes(bits, blk, out, lt, dt)
        else:
            raise InflateError('reserved block type 3')
        blk.end_bit = bits.pos
        blk.out = bytes(out[blk.out_start:])
        blocks.append(blk)
    a = (bits.pos + 7) >> 3
    if len(body) < a + 4:
        raise InflateError('truncated stream')
    if int.from_bytes(body[a:a + 4], 'big') != zlib.adler32(bytes(out)):
        raise InflateError('Adler-32 mismatch')
    if len(body) != a + 4:
        raise InflateError(f'{len(body) - a - 4} bytes after the stream')
    return blocks


def replay(tokens, history=b''):
    """The bytes a token list decodes to, after ``history`` (the window before it)."""
    out = bytearray(history)
    for t in tokens:
        if isinstance(t, tuple):
            length, dist = t
            for _ in range(length):
                out.append(out[-dist])
        elif t != EOB:
            out.append(t)
    return bytes(out[len(history):])


def histograms(tokens):
    """(literal / length histogram [286] with EOB counted once per EOB token, distance histogram [30])."""
    ll, d = [0] * 286, [0] * 30
    for t in tokens:
        if isinstance(t, tuple):
            ll[257 + _LEN_CODE[t[0]]] += 1
            d[_DIST_CODE[t[1]]] += 1
        else:
            ll[t] += 1
    return ll, d


def at_least_two(f):
    """The encoder's rule for a code that must be complete with >= 2 codes: no non-zero count -> f[0] = f[1] = 1; one
    non-zero count -> the first of f[0], f[1] that is zero becomes 1.  Returns a new list."""
    f = list(f)
    nz = sum(x > 0 for x in f)
    if nz == 0:
        f[0] = f[1] = 1
    elif nz == 1:
        f[1 if f[0] else 0] = 1
    return f


def optimal_limited_cost(freq, maxbits):
    """min sum f_i l_i over prefix codes of the symbols with f_i > 0 and 1 <= l_i <= maxbits (package-merge).  One
    symbol costs its frequency (deflate has no 0-bit code); more than 2^maxbits symbols raise ValueError."""
    w = sorted(int(f) for f in freq if f > 0)
    m = len(w)
    if m <= 1:
        return sum(w)
    if m > 1 << maxbits:
        raise ValueError(f'{m} symbols do not fit in codes of <= {maxbits} bits')
    items = list(w)
    for _ in range(maxbits - 1):              # the lists of levels maxbits - 1 .. 1: leaves merged with packages
        packages = [items[2 * i] + items[2 * i + 1] for i in range(len(items) // 2)]
        items = sorted(w + packages)
    return sum(items[:2 * m - 2])


def huffman_cost(freq):
    """min sum f_i l_i over prefix codes of the symbols with f_i > 0, without a length limit (Huffman)."""
    h = sorted(int(f) for f in freq if f > 0)
    if len(h) <= 1:
        return sum(h)
    heapq.heapify(h)
    cost = 0
    while len(h) > 1:
        s = heapq.heappop(h) + heapq.heappop(h)
        cost += s
        heapq.heappush(h, s)
    return cost


def code_cost(freq, lens):
    return sum(int(f) * int(l) for f, l in zip(freq, lens))
