// k4_png.cu -- PNG files of uint8 RGB frames encoded on the device (k4_png_encode), for run_sr.py --render_test's
// imageio.imwrite of every SR / LR frame (run_sr.py:171-175, 1390-1396).
//
// The file: signature, IHDR (W, H, depth 8, colour type 2, no interlace), one IDAT chunk holding the zlib stream, IEND.
// Stages, all on the caller's stream:
//   png_filter_kernel    one warp per row: the five PNG filters, the one with the least sum of |byte as int8| (libpng's
//                        heuristic; ties to the lowest type), written as [type | filtered row] into the filtered stream
//   png_match_kernel     one CTA per segment of K4_PNG_SEG bytes of the filtered stream: for every position the longest
//                        match among a hash-table candidate (the latest earlier position of the window with the same
//                        3-byte hash, taken before each 1024-position chunk), the previous lane of the warp with the same
//                        hash, and the fixed distances 1, 2, 3, 4, 6 and one filtered row.  Matches reach up to 32 KiB
//                        before the segment's start and end at the segment's end.
//   png_encode_kernel    one CTA per segment: lazy parse (one thread), symbol histograms, code lengths limited to 15
//                        (7 for the code-length code) by package-merge, one dynamic-Huffman block written in parallel
//                        (per-thread bit counts, a block scan, atomicOr into shared memory), or a stored block when the
//                        dynamic one is not smaller.  A dynamic segment other than the last ends with an empty stored
//                        block, so every segment starts on a byte boundary.  The segment's Adler-32 pair too.
//   png_join_kernel      one CTA: byte offsets of the segments (a scan), the Adler-32 combined over the segments, the
//                        container's bytes around the deflate data
//   png_copy_kernel      the segments to their offsets
//   png_crc_kernel       CRC-32 of 1 KiB pieces of the IDAT chunk's type and data
//   png_crc_join_kernel  the pieces' CRCs joined by the GF(2) shift x^(8 len) mod P (zlib's crc32_combine)
// Everything is a fixed function of the frame: the table inserts are atomicMax of positions, the histograms integer
// atomics, and every choice has a tie rule.
#include "k4_internal.cuh"

namespace {

constexpr int SEG = K4_PNG_SEG;           // filtered bytes per segment (one CTA each)
constexpr int NT = 1024;                  // threads of the match and encode kernels
constexpr int PER_T = SEG / NT;           // positions per thread in the encoder
constexpr int HBITS = 14;                 // hash table: 2^14 latest positions per window
constexpr int WIN = 32768;
constexpr int MAXM = 258;
constexpr int CRC_PIECE = 1024;
constexpr int OUT_WORDS = (SEG + 64) / 4; // a segment's dynamic block is kept only below 5 + SEG bytes
constexpr int HDR = 43;                   // signature, IHDR, IDAT length and type, zlib header
constexpr uint32_t ADLER_MOD = 65521u;
constexpr uint32_t CRC_POLY = 0xedb88320u;

static_assert(SEG % NT == 0 && SEG <= 65535, "a stored segment is one stored block");

static_assert(PER_T == 32, "the encoder's start bitmap holds one word per thread");

struct PngWs {
    size_t filt, best, segout, seglen, segoff, segadl, crc, misc, total;
};

__host__ __device__ inline int64_t png_n(int64_t H, int64_t W) { return H * (1 + 3 * W); }
__host__ __device__ inline int64_t png_nseg(int64_t n) { return (n + SEG - 1) / SEG; }
inline size_t up256(size_t x) { return (x + 255) & ~size_t(255); }

PngWs png_ws_layout(int64_t H, int64_t W) {
    const int64_t n = png_n(H, W), ns = png_nseg(n);
    const int64_t ncrc = (n + 5 * ns + 63) / CRC_PIECE + 2;
    PngWs L;
    size_t o = 0;
    L.filt = o;   o += up256(n + 16);
    L.best = o;   o += up256(n * 4);
    L.segout = o; o += up256(ns * (size_t)(OUT_WORDS * 4));
    L.seglen = o; o += up256(ns * 4);
    L.segoff = o; o += up256(ns * 8);
    L.segadl = o; o += up256(ns * 4);
    L.crc = o;    o += up256(ncrc * 4);
    L.misc = o;   o += 256;
    L.total = o;
    return L;
}

// ---- CRC-32 (reflected, polynomial 0xedb88320) ------------------------------------------------------
__host__ __device__ inline uint32_t crc_byte_update(uint32_t c, uint8_t b) {
    c ^= b;
    for (int k = 0; k < 8; ++k) c = c & 1 ? (c >> 1) ^ CRC_POLY : c >> 1;
    return c;
}
// a * b mod P in the reflected representation (bit 31 is x^0)
__device__ inline uint32_t gf2_mulmod(uint32_t a, uint32_t b) {
    uint32_t m = 1u << 31, p = 0;
    if (!a) return 0;
    for (;;) {
        if (a & m) {
            p ^= b;
            if ((a & (m - 1)) == 0) break;
        }
        m >>= 1;
        b = b & 1 ? (b >> 1) ^ CRC_POLY : b >> 1;
    }
    return p;
}
// x^(8 n) mod P: squares of x^8 picked by the bits of n
__device__ inline uint32_t gf2_x8n(int64_t n) {
    uint32_t p = 1u << 31, sq = 1u << 23;            // x^0, x^8
    while (n) {
        if (n & 1) p = gf2_mulmod(sq, p);
        sq = gf2_mulmod(sq, sq);
        n >>= 1;
    }
    return p;
}
// CRC of A || B from CRC(A), CRC(B) and |B|
__device__ inline uint32_t crc_join(uint32_t ca, uint32_t cb, int64_t lb) { return gf2_mulmod(gf2_x8n(lb), ca) ^ cb; }

// ---- Adler-32 ----------------------------------------------------------------------------------------
__device__ inline uint32_t adler_join(uint32_t a1, uint32_t a2, int64_t len2) {
    const uint32_t rem = (uint32_t)(len2 % ADLER_MOD);
    uint32_t s1 = a1 & 0xffff;
    uint32_t s2 = (uint32_t)(((uint64_t)rem * s1) % ADLER_MOD);
    s1 += (a2 & 0xffff) + ADLER_MOD - 1;
    s2 += (a1 >> 16) + (a2 >> 16) + ADLER_MOD - rem;
    if (s1 >= ADLER_MOD) s1 -= ADLER_MOD;
    if (s1 >= ADLER_MOD) s1 -= ADLER_MOD;
    if (s2 >= 2 * ADLER_MOD) s2 -= 2 * ADLER_MOD;
    if (s2 >= ADLER_MOD) s2 -= ADLER_MOD;
    return s1 | (s2 << 16);
}

// ---- deflate's length and distance codes (RFC 1951 3.2.5), from the bit patterns of len - 3 and d - 1 ----
// the code-length code's symbols in the order of the block header
__constant__ uint8_t c_cl_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

__device__ inline int len_code(int len) {             // 3..258 -> 0..28
    const int x = len - 3;
    if (len == 258) return 28;
    if (x < 8) return x;
    const int b = 31 - __clz(x);
    return 4 * (b - 1) + ((x >> (b - 2)) & 3);
}
__device__ inline int len_extra(int lc) { return lc < 8 || lc == 28 ? 0 : (lc - 4) >> 2; }
__device__ inline int dist_code(int d) {              // 1..32768 -> 0..29
    const int x = d - 1;
    if (x < 4) return x;
    const int b = 31 - __clz(x);
    return 2 * b + ((x >> (b - 1)) & 1);
}
__device__ inline int dist_extra(int dc) { return dc < 4 ? 0 : (dc - 2) >> 1; }

// ---- filtering --------------------------------------------------------------------------------------
__device__ inline int paeth(int a, int b, int c) {
    const int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
    return pa <= pb && pa <= pc ? a : pb <= pc ? b : c;
}
__device__ inline uint8_t filt_byte(int f, int x, int a, int b, int c) {
    switch (f) {
        case 0: return (uint8_t)x;
        case 1: return (uint8_t)(x - a);
        case 2: return (uint8_t)(x - b);
        case 3: return (uint8_t)(x - ((a + b) >> 1));
        default: return (uint8_t)(x - paeth(a, b, c));
    }
}
__device__ inline int sabs8(uint8_t v) { return v < 128 ? v : 256 - v; }

__global__ void __launch_bounds__(256) png_filter_kernel(const uint8_t* __restrict__ rgb, int H, int W,
                                                         uint8_t* __restrict__ filt) {
    const int lane = threadIdx.x & 31;
    const int y = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (y >= H) return;
    const int rb = 3 * W;
    const uint8_t* cur = rgb + (size_t)y * rb;
    const uint8_t* prv = y ? cur - rb : nullptr;
    int s[5] = {0, 0, 0, 0, 0};
    for (int i = lane; i < rb; i += 32) {
        const int x = cur[i], a = i >= 3 ? cur[i - 3] : 0, b = prv ? prv[i] : 0, c = prv && i >= 3 ? prv[i - 3] : 0;
#pragma unroll
        for (int f = 0; f < 5; ++f) s[f] += sabs8(filt_byte(f, x, a, b, c));
    }
#pragma unroll
    for (int f = 0; f < 5; ++f)
#pragma unroll
        for (int o = 16; o; o >>= 1) s[f] += __shfl_xor_sync(0xffffffffu, s[f], o);
    int best = 0;
#pragma unroll
    for (int f = 1; f < 5; ++f)
        if (s[f] < s[best]) best = f;
    uint8_t* out = filt + (size_t)y * (rb + 1);
    if (lane == 0) out[0] = (uint8_t)best;
    for (int i = lane; i < rb; i += 32) {
        const int x = cur[i], a = i >= 3 ? cur[i - 3] : 0, b = prv ? prv[i] : 0, c = prv && i >= 3 ? prv[i - 3] : 0;
        out[1 + i] = filt_byte(best, x, a, b, c);
    }
}

// ---- match finding ----------------------------------------------------------------------------------
__device__ inline uint32_t win_word(const uint32_t* w, int i) {   // 4 bytes at byte index i (little-endian)
    const int k = i >> 2, r = (i & 3) * 8;
    return __funnelshift_r(w[k], w[k + 1], r);
}
__device__ inline int match_len(const uint32_t* w, int c, int p, int maxlen) {
    int k = 0;
    while (k < maxlen) {
        const uint32_t x = win_word(w, c + k) ^ win_word(w, p + k);
        if (x) return min(maxlen, k + ((__ffs(x) - 1) >> 3));
        k += 4;
    }
    return maxlen;
}
__device__ inline uint32_t hash3(uint32_t v) { return ((v & 0xffffffu) * 2654435761u) >> (32 - HBITS); }

__global__ void __launch_bounds__(NT) png_match_kernel(const uint8_t* __restrict__ filt, int64_t n, int stride,
                                                      uint32_t* __restrict__ best) {
    extern __shared__ __align__(16) uint32_t sm[];
    int* table = (int*)sm;                                      // [1 << HBITS] window index of the latest insert
    uint32_t* w = sm + (1 << HBITS);                            // the window's bytes, [WIN + SEG + 16]
    const int64_t s0 = (int64_t)blockIdx.x * SEG, s1 = min(n, s0 + SEG), w0 = max((int64_t)0, s0 - WIN);
    const int wn = (int)(s1 - w0), seg_lo = (int)(s0 - w0);
    for (int i = threadIdx.x; i < (1 << HBITS); i += NT) table[i] = -1;
    uint8_t* wb = (uint8_t*)w;
    for (int i = threadIdx.x; i < ((wn + 8 + 3) & ~3); i += NT) wb[i] = i < wn ? filt[w0 + i] : 0;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    for (int base = 0; base < wn; base += NT) {
        const int p = base + threadIdx.x;
        const bool valid = p + 3 <= wn;
        const uint32_t h = valid ? hash3(win_word(w, p)) : 0;
        const uint32_t grp = __match_any_sync(0xffffffffu, valid ? h : 0x80000000u | lane);
        const uint32_t lower = grp & ((1u << lane) - 1);
        const int c_warp = valid && lower ? p - lane + (31 - __clz(lower)) : -1;
        const int c_tab = valid ? table[h] : -1;
        __syncthreads();
        if (valid) atomicMax(&table[h], p);
        if (p >= seg_lo && p < wn) {
            uint32_t m = 0;
            if (valid) {
                const int maxlen = min(MAXM, wn - p);
                int bl = 2, bd = 0;
                const int cands[8] = {c_warp, c_tab, p - 1, p - 2, p - 3, p - 4, p - 6, p - stride};
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    const int c = cands[k];
                    if (c < 0 || c >= p || p - c > WIN) continue;
                    const int l = match_len(w, c, p, maxlen);
                    if (l > bl || (l == bl && l >= 3 && p - c < bd)) { bl = l; bd = p - c; }
                }
                if (bl >= 3 && !(bl == 3 && bd > 4096)) m = ((uint32_t)bl << 16) | (uint32_t)(bd - 1);
            }
            best[w0 + p] = m;
        }
        __syncthreads();
    }
}

// ---- Huffman code lengths ---------------------------------------------------------------------------
constexpr int MAXSYM = 286;
struct HuffSmem {
    int ll_f[MAXSYM], d_f[30], cl_f[19];
    uint8_t ll_l[MAXSYM], d_l[30], cl_l[19];
    uint16_t ll_c[MAXSYM], d_c[30], cl_c[19];
    uint16_t sorted[MAXSYM];
    uint32_t wa[2 * MAXSYM], wb[2 * MAXSYM];
    uint8_t flags[16][2 * MAXSYM];
    int bl_cnt[16], bl_next[16];
    uint16_t rle_sym[MAXSYM + 30];
    uint8_t rle_x[MAXSYM + 30];
    int n_rle, n_rle_ll, m;
    int hlit, hdist, hclen;
    uint32_t hdr_bits, total_bits, dyn;
    uint64_t adl_a, adl_b;
};

// Length-limited Huffman code lengths of freq[0..n) (package-merge).  All threads call it.
__device__ void huff_lengths(const int* freq, int n, int maxbits, uint8_t* len, HuffSmem& s) {
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        len[i] = 0;
        const int f = freq[i];
        if (f > 0) {
            int r = 0;
            for (int j = 0; j < n; ++j) r += freq[j] > 0 && (freq[j] < f || (freq[j] == f && j < i));
            s.sorted[r] = (uint16_t)i;
        }
    }
    if (threadIdx.x == 0) {
        int m = 0;
        for (int j = 0; j < n; ++j) m += freq[j] > 0;
        s.m = m;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const int m = s.m;
        if (m == 1) len[s.sorted[0]] = 1;
        if (m >= 2) {
            uint32_t* cur = s.wa;
            uint32_t* nxt = s.wb;
            for (int i = 0; i < m; ++i) cur[i] = (uint32_t)freq[s.sorted[i]];
            int cnt = m;
            for (int l = 2; l <= maxbits; ++l) {
                const int np = cnt / 2;
                int i = 0, k = 0, o = 0;
                while (i < m || k < np) {
                    const uint32_t lf = i < m ? (uint32_t)freq[s.sorted[i]] : 0xffffffffu;
                    const uint32_t pk = k < np ? cur[2 * k] + cur[2 * k + 1] : 0xffffffffu;
                    if (i < m && (k >= np || lf <= pk)) { nxt[o] = lf; s.flags[l][o] = 1; ++i; }
                    else { nxt[o] = pk; s.flags[l][o] = 0; ++k; }
                    ++o;
                }
                uint32_t* t = cur; cur = nxt; nxt = t;
                cnt = o;
            }
            int k = 2 * m - 2;
            for (int l = maxbits; l >= 2; --l) {
                int nl = 0;
                for (int j = 0; j < k; ++j) nl += s.flags[l][j];
                for (int r = 0; r < nl; ++r) ++len[s.sorted[r]];
                k = 2 * (k - nl);
            }
            for (int r = 0; r < k; ++r) ++len[s.sorted[r]];
        }
    }
    __syncthreads();
}

// canonical codes, bit-reversed for deflate's LSB-first stream (one thread)
__device__ void huff_codes(const uint8_t* len, int n, uint16_t* code, int* cnt, int* next) {
    for (int b = 0; b < 16; ++b) cnt[b] = 0;
    for (int i = 0; i < n; ++i) ++cnt[len[i]];
    cnt[0] = 0;
    int c = 0;
    for (int b = 1; b < 16; ++b) { c = (c + cnt[b - 1]) << 1; next[b] = c; }
    for (int i = 0; i < n; ++i)
        if (len[i]) code[i] = (uint16_t)(__brev((uint32_t)next[len[i]]++) >> (32 - len[i]));
}

// run-length code of lens[0..n) with the code-length code's symbols 16 / 17 / 18 (RFC 1951 3.2.7), appended to s.rle_*
__device__ void rle_lengths(const uint8_t* lens, int n, HuffSmem& s) {
    int i = 0;
    while (i < n) {
        const int v = lens[i];
        int run = 1;
        while (i + run < n && lens[i + run] == v) ++run;
        i += run;
        if (v == 0) {
            while (run >= 11) { const int r = min(run, 138); s.rle_sym[s.n_rle] = 18; s.rle_x[s.n_rle++] = (uint8_t)(r - 11); run -= r; }
            if (run >= 3) { s.rle_sym[s.n_rle] = 17; s.rle_x[s.n_rle++] = (uint8_t)(run - 3); run = 0; }
        } else {
            s.rle_sym[s.n_rle] = (uint16_t)v; s.rle_x[s.n_rle++] = 0; --run;
            while (run >= 3) { const int r = min(run, 6); s.rle_sym[s.n_rle] = 16; s.rle_x[s.n_rle++] = (uint8_t)(r - 3); run -= r; }
        }
        while (run-- > 0) { s.rle_sym[s.n_rle] = (uint16_t)v; s.rle_x[s.n_rle++] = 0; }
    }
}

__device__ inline void at_least_two(int* f, int n) {      // a complete code of >= 2 symbols (one thread)
    int nz = 0;
    for (int i = 0; i < n; ++i) nz += f[i] > 0;
    if (nz == 0) f[0] = f[1] = 1;
    else if (nz == 1) f[f[0] ? 1 : 0] = 1;
}

__device__ inline void put_bits(uint32_t* out, uint32_t pos, uint32_t v, int nb) {   // nb <= 32, LSB first
    if (!nb) return;
    const uint32_t w = pos >> 5, sh = pos & 31;
    atomicOr(&out[w], v << sh);
    if (sh + nb > 32) atomicOr(&out[w + 1], v >> (32 - sh));
}

__device__ inline uint32_t block_excl_scan(uint32_t v, uint32_t* tmp, uint32_t* total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) tmp[wid] = x;
    __syncthreads();
    if (wid == 0) {
        uint32_t t = lane < (int)(blockDim.x >> 5) ? tmp[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, t, o); if (lane >= o) t += y; }
        tmp[lane] = t;
    }
    __syncthreads();
    const uint32_t r = x - v + (wid ? tmp[wid - 1] : 0);
    *total = tmp[(blockDim.x >> 5) - 1];
    __syncthreads();
    return r;
}

// bits of the token at local position p (its symbols already counted)
__device__ inline uint32_t token_bits(uint32_t m, uint8_t lit, const HuffSmem& s) {
    if (!m) return s.ll_l[lit];
    const int len = m >> 16, d = (m & 0xffff) + 1;
    const int lc = len_code(len), dc = dist_code(d);
    return s.ll_l[257 + lc] + len_extra(lc) + s.d_l[dc] + dist_extra(dc);
}

__global__ void __launch_bounds__(NT, 1) png_encode_kernel(const uint8_t* __restrict__ filt, int64_t n,
                                                          const uint32_t* __restrict__ best_g, uint8_t* __restrict__ segout,
                                                          uint32_t* __restrict__ seglen, uint32_t* __restrict__ segadl) {
    extern __shared__ __align__(16) uint32_t sm[];
    uint32_t* best = sm;                                        // [SEG]
    uint32_t* out = best + SEG;                                 // [OUT_WORDS + 2]
    uint32_t* starts = out + OUT_WORDS + 2;                     // [SEG / 32]
    uint32_t* tmp = starts + SEG / 32;                          // [32]
    __shared__ HuffSmem s;
    const int seg = blockIdx.x, nseg = gridDim.x, t = threadIdx.x;
    const int64_t s0 = (int64_t)seg * SEG;
    const int L = (int)min((int64_t)SEG, n - s0);
    const bool last = seg == nseg - 1;
    const uint8_t* src = filt + s0;
    for (int i = t; i < L; i += NT) best[i] = best_g[s0 + i];
    for (int i = t; i < OUT_WORDS + 2; i += NT) out[i] = 0;
    for (int i = t; i < SEG / 32; i += NT) starts[i] = 0;
    for (int i = t; i < MAXSYM; i += NT) s.ll_f[i] = 0;
    if (t < 30) s.d_f[t] = 0;
    if (t < 19) s.cl_f[t] = 0;
    if (t == 0) { s.n_rle = 0; s.adl_a = 0; s.adl_b = 0; }
    __syncthreads();

    // Adler-32 of the segment: a = 1 + sum d, b = L + sum (L - i) d_i
    {
        uint64_t a = 0, b = 0;
        for (int i = t; i < L; i += NT) { const uint32_t d = src[i]; a += d; b += (uint64_t)(L - i) * d; }
#pragma unroll
        for (int o = 16; o; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); b += __shfl_xor_sync(0xffffffffu, b, o); }
        if ((t & 31) == 0) { atomicAdd((unsigned long long*)&s.adl_a, a); atomicAdd((unsigned long long*)&s.adl_b, b); }
    }

    // lazy parse: a match is taken unless the next position has a longer one
    if (t == 0) {
        int p = 0;
        while (p < L) {
            const uint32_t m = best[p];
            const int len = m >> 16;
            starts[p >> 5] |= 1u << (p & 31);
            if (len >= 3 && !(p + 1 < L && (best[p + 1] >> 16) > (uint32_t)len)) {
                p += len;
            } else {
                best[p] = 0;
                ++p;
            }
        }
    }
    __syncthreads();
    if (t == 0) segadl[seg] = (uint32_t)((1 + s.adl_a) % ADLER_MOD) | ((uint32_t)((L + s.adl_b) % ADLER_MOD) << 16);

    // symbol histograms
    const uint32_t st = starts[t];
    for (int j = 0; j < PER_T; ++j) {
        const int p = t * PER_T + j;
        if (p >= L || !((st >> j) & 1)) continue;
        const uint32_t m = best[p];
        if (!m) atomicAdd(&s.ll_f[src[p]], 1);
        else {
            atomicAdd(&s.ll_f[257 + len_code(m >> 16)], 1);
            atomicAdd(&s.d_f[dist_code((m & 0xffff) + 1)], 1);
        }
    }
    __syncthreads();
    if (t == 0) {
        s.ll_f[256] = 1;
        at_least_two(s.d_f, 30);             // two distance codes at least: one code alone would be a 0-bit code
    }
    __syncthreads();
    huff_lengths(s.ll_f, MAXSYM, 15, s.ll_l, s);
    huff_lengths(s.d_f, 30, 15, s.d_l, s);
    if (t == 0) {
        huff_codes(s.ll_l, MAXSYM, s.ll_c, s.bl_cnt, s.bl_next);
        huff_codes(s.d_l, 30, s.d_c, s.bl_cnt, s.bl_next);
        int hl = MAXSYM;
        while (hl > 257 && !s.ll_l[hl - 1]) --hl;
        int hd = 30;
        while (hd > 1 && !s.d_l[hd - 1]) --hd;
        s.hlit = hl;
        s.hdist = hd;
        rle_lengths(s.ll_l, hl, s);
        s.n_rle_ll = s.n_rle;
        rle_lengths(s.d_l, hd, s);
        for (int i = 0; i < s.n_rle; ++i) ++s.cl_f[s.rle_sym[i]];
        at_least_two(s.cl_f, 19);
    }
    __syncthreads();
    huff_lengths(s.cl_f, 19, 7, s.cl_l, s);

    // per-thread token bits and their offsets
    uint32_t mybits = 0;
    for (int j = 0; j < PER_T; ++j) {
        const int p = t * PER_T + j;
        if (p < L && ((st >> j) & 1)) mybits += token_bits(best[p], src[p], s);
    }
    uint32_t data_bits;
    const uint32_t my_off = block_excl_scan(mybits, tmp, &data_bits);
    if (t == 0) {
        huff_codes(s.cl_l, 19, s.cl_c, s.bl_cnt, s.bl_next);
        int hc = 19;
        while (hc > 4 && !s.cl_l[c_cl_order[hc - 1]]) --hc;
        s.hclen = hc;
        uint32_t hb = 3 + 5 + 5 + 4 + 3 * hc;
        for (int i = 0; i < s.n_rle; ++i) {
            const int y = s.rle_sym[i];
            hb += s.cl_l[y] + (y == 16 ? 2 : y == 17 ? 3 : y == 18 ? 7 : 0);
        }
        s.hdr_bits = hb;
        const uint32_t bits = hb + data_bits + s.ll_l[256] + (last ? 0 : 3);
        const uint32_t bytes = (bits + 7) / 8 + (last ? 0 : 4);
        s.dyn = bytes < (uint32_t)(5 + L);
        s.total_bits = bits;
    }
    __syncthreads();
    uint8_t* dst = segout + (size_t)seg * (OUT_WORDS * 4);
    if (!s.dyn) {
        if (t == 0) {
            dst[0] = last ? 1 : 0;
            dst[1] = (uint8_t)L; dst[2] = (uint8_t)(L >> 8);
            dst[3] = (uint8_t)~L; dst[4] = (uint8_t)(~L >> 8);
            seglen[seg] = 5 + L;
        }
        for (int i = t; i < L; i += NT) dst[5 + i] = src[i];
        return;
    }
    if (t == 0) {
        uint32_t b = 0;
        put_bits(out, b, last ? 5 : 4, 3); b += 3;                // BFINAL, BTYPE = 10
        put_bits(out, b, s.hlit - 257, 5); b += 5;
        put_bits(out, b, s.hdist - 1, 5); b += 5;
        put_bits(out, b, s.hclen - 4, 4); b += 4;
        for (int i = 0; i < s.hclen; ++i) { put_bits(out, b, s.cl_l[c_cl_order[i]], 3); b += 3; }
        for (int i = 0; i < s.n_rle; ++i) {
            const int y = s.rle_sym[i];
            put_bits(out, b, s.cl_c[y], s.cl_l[y]); b += s.cl_l[y];
            const int xb = y == 16 ? 2 : y == 17 ? 3 : y == 18 ? 7 : 0;
            put_bits(out, b, s.rle_x[i], xb); b += xb;
        }
        const uint32_t e = s.hdr_bits + data_bits;
        put_bits(out, e, s.ll_c[256], s.ll_l[256]);            // end of block; a sync flush's 3 zero bits follow
    }
    uint32_t b = s.hdr_bits + my_off;
    for (int j = 0; j < PER_T; ++j) {
        const int p = t * PER_T + j;
        if (p >= L || !((st >> j) & 1)) continue;
        const uint32_t m = best[p];
        if (!m) {
            const int y = src[p];
            put_bits(out, b, s.ll_c[y], s.ll_l[y]); b += s.ll_l[y];
        } else {
            const int len = m >> 16, d = (m & 0xffff) + 1, lc = len_code(len), dc = dist_code(d);
            const int le = len_extra(lc), de = dist_extra(dc);
            put_bits(out, b, s.ll_c[257 + lc], s.ll_l[257 + lc]); b += s.ll_l[257 + lc];
            put_bits(out, b, (len - 3) & ((1 << le) - 1), le); b += le;
            put_bits(out, b, s.d_c[dc], s.d_l[dc]); b += s.d_l[dc];
            put_bits(out, b, (d - 1) & ((1 << de) - 1), de); b += de;
        }
    }
    __syncthreads();
    const uint32_t nbytes = (s.total_bits + 7) / 8;
    const uint8_t* ob = (const uint8_t*)out;
    for (uint32_t i = t; i < nbytes; i += NT) dst[i] = ob[i];
    if (!last && t < 4) dst[nbytes + t] = t < 2 ? 0x00 : 0xff;   // LEN = 0, NLEN = 0xffff
    if (t == 0) seglen[seg] = nbytes + (last ? 0 : 4);
}

// ---- container ----------------------------------------------------------------------------------------
struct PngHead {
    uint8_t b[33];                        // signature and IHDR chunk
};

__device__ inline void put_be32(uint8_t* p, uint32_t v) {
    p[0] = (uint8_t)(v >> 24); p[1] = (uint8_t)(v >> 16); p[2] = (uint8_t)(v >> 8); p[3] = (uint8_t)v;
}

__global__ void __launch_bounds__(NT) png_join_kernel(const uint32_t* __restrict__ seglen, const uint32_t* __restrict__ segadl,
                                                     int64_t n, int64_t nseg, int64_t* __restrict__ segoff, int64_t* __restrict__ misc,
                                                     const __grid_constant__ PngHead head, uint8_t* __restrict__ out,
                                                     int64_t* __restrict__ d_len) {
    __shared__ uint32_t tmp[32];
    __shared__ int64_t carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int64_t b0 = 0; b0 < nseg; b0 += NT) {
        const int64_t i = b0 + threadIdx.x;
        const uint32_t v = i < nseg ? seglen[i] : 0;
        uint32_t tot;
        const uint32_t ex = block_excl_scan(v, tmp, &tot);
        if (i < nseg) segoff[i] = carry + ex;
        __syncthreads();
        if (threadIdx.x == 0) carry += tot;
        __syncthreads();
    }
    if (threadIdx.x != 0) return;
    const int64_t D = carry;
    uint32_t adl = 1;
    for (int64_t i = 0; i < nseg; ++i) adl = adler_join(adl, segadl[i], min((int64_t)SEG, n - i * SEG));
    misc[0] = D;
    for (int i = 0; i < 33; ++i) out[i] = head.b[i];
    put_be32(out + 33, (uint32_t)(D + 6));
    out[37] = 'I'; out[38] = 'D'; out[39] = 'A'; out[40] = 'T';
    out[41] = 0x78; out[42] = 0x9c;
    put_be32(out + HDR + D, adl);
    uint8_t* e = out + HDR + D + 8;
    put_be32(e, 0);
    e[4] = 'I'; e[5] = 'E'; e[6] = 'N'; e[7] = 'D';
    put_be32(e + 8, 0xae426082u);
    *d_len = HDR + D + 20;
}

__global__ void __launch_bounds__(256) png_copy_kernel(const uint8_t* __restrict__ segout, const uint32_t* __restrict__ seglen,
                                                      const int64_t* __restrict__ segoff, uint8_t* __restrict__ out) {
    const int s = blockIdx.x;
    const uint8_t* src = segout + (size_t)s * (OUT_WORDS * 4);
    uint8_t* dst = out + HDR + segoff[s];
    const uint32_t len = seglen[s];
    for (uint32_t i = threadIdx.x; i < len; i += blockDim.x) dst[i] = src[i];
}

// CRC of the IDAT chunk's type and data, out[37, 47 + D), in pieces of CRC_PIECE bytes
__global__ void __launch_bounds__(256) png_crc_kernel(const uint8_t* __restrict__ out, const int64_t* __restrict__ misc,
                                                     int64_t npieces, uint32_t* __restrict__ crc) {
    __shared__ uint32_t tab[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) {
        uint32_t c = i;
        for (int k = 0; k < 8; ++k) c = c & 1 ? (c >> 1) ^ CRC_POLY : c >> 1;
        tab[i] = c;
    }
    __syncthreads();
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= npieces) return;
    const int64_t len = misc[0] + 10;
    const int64_t a = min(len, k * CRC_PIECE), b = min(len, a + CRC_PIECE);
    uint32_t c = 0xffffffffu;
    for (int64_t i = a; i < b; ++i) c = tab[(c ^ out[37 + i]) & 0xff] ^ (c >> 8);
    crc[k] = c ^ 0xffffffffu;
}

__global__ void __launch_bounds__(NT) png_crc_join_kernel(const uint32_t* __restrict__ crc, const int64_t* __restrict__ misc,
                                                         uint8_t* __restrict__ out) {
    __shared__ uint32_t c_s[NT];
    __shared__ int64_t l_s[NT];
    const int64_t len = misc[0] + 10;
    const int64_t np = (len + CRC_PIECE - 1) / CRC_PIECE;
    const int64_t per = (np + NT - 1) / NT;
    const int64_t k0 = min(np, threadIdx.x * per), k1 = min(np, k0 + per);
    const uint32_t shift = gf2_x8n(CRC_PIECE);
    uint32_t c = 0;
    int64_t l = 0;
    for (int64_t k = k0; k < k1; ++k) {
        const int64_t lk = min((int64_t)CRC_PIECE, len - k * CRC_PIECE);
        c = (lk == CRC_PIECE ? gf2_mulmod(shift, c) : gf2_mulmod(gf2_x8n(lk), c)) ^ crc[k];
        l += lk;
    }
    c_s[threadIdx.x] = c;
    l_s[threadIdx.x] = l;
    __syncthreads();
    for (int w = 1; w < NT; w <<= 1) {
        uint32_t cn = 0;
        int64_t ln = 0;
        const int i = threadIdx.x;
        const bool act = (i % (2 * w)) == 0 && i + w < NT;
        if (act) { cn = l_s[i + w] ? crc_join(c_s[i], c_s[i + w], l_s[i + w]) : c_s[i]; ln = l_s[i] + l_s[i + w]; }
        __syncthreads();
        if (act) { c_s[i] = cn; l_s[i] = ln; }
        __syncthreads();
    }
    if (threadIdx.x == 0) put_be32(out + 47 + misc[0], c_s[0]);
}

int launch_error(const char* where) {
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { k4_set_cuda_error(e, where); return K4_ERR_CUDA; }
    return K4_OK;
}

// k4_testing_png_code_lengths: huff_lengths on a caller's histogram, one CTA of NT threads as in png_encode_kernel.
// Histograms package-merge cannot code (more non-zero counts than 2^maxbits, or a total that overflows its 32-bit item
// weights) get 0xff for every length instead.
__global__ void __launch_bounds__(NT) png_code_lengths_kernel(const int32_t* __restrict__ freq, int n, int maxbits,
                                                             uint8_t* __restrict__ len) {
    __shared__ HuffSmem s;
    __shared__ int ok;
    for (int i = threadIdx.x; i < n; i += NT) s.ll_f[i] = freq[i];
    __syncthreads();
    if (threadIdx.x == 0) {
        int m = 0;
        int64_t tot = 0;
        for (int i = 0; i < n; ++i)
            if (s.ll_f[i] > 0) { ++m; tot += s.ll_f[i]; }
        ok = m <= (1 << maxbits) && tot < 0x7fffffff;
    }
    __syncthreads();
    if (!ok) {
        for (int i = threadIdx.x; i < n; i += NT) len[i] = 0xff;
        return;
    }
    huff_lengths(s.ll_f, n, maxbits, s.ll_l, s);
    for (int i = threadIdx.x; i < n; i += NT) len[i] = s.ll_l[i];
}

constexpr size_t MATCH_SMEM = (size_t)(1 << HBITS) * 4 + (WIN + SEG + 16);
constexpr size_t ENC_SMEM = (size_t)(SEG + OUT_WORDS + 2 + SEG / 32 + 32) * 4;

bool png_shape_ok(int64_t H, int64_t W) {
    if (H < 1 || W < 1 || H > (1 << 30) || W > (1 << 28)) return false;
    return png_n(H, W) + 5 * png_nseg(png_n(H, W)) + 63 <= 0x7fffffff;    // one IDAT chunk: length < 2^31
}

}  // namespace

extern "C" {

size_t k4_png_encode_bound(int64_t H, int64_t W) {
    if (!png_shape_ok(H, W)) return 0;
    const int64_t n = png_n(H, W);
    return (size_t)(n + 5 * png_nseg(n) + HDR + 20);
}

size_t k4_png_workspace_bytes(int64_t H, int64_t W) {
    if (!png_shape_ok(H, W)) return 0;
    return png_ws_layout(H, W).total;
}

int k4_png_encode(const uint8_t* d_rgb, int64_t H, int64_t W, uint8_t* d_out, size_t out_capacity, int64_t* d_len,
                  void* d_workspace, size_t workspace_bytes, k4_stream_t stream) {
    if (!d_rgb || !d_out || !d_len || !d_workspace) return K4_ERR_INVALID_ARG;
    if (!png_shape_ok(H, W)) return K4_ERR_INVALID_ARG;
    if (out_capacity < k4_png_encode_bound(H, W) || workspace_bytes < k4_png_workspace_bytes(H, W)) return K4_ERR_INVALID_ARG;
    if ((uintptr_t)d_workspace % 256 || (uintptr_t)d_len % 8) return K4_ERR_INVALID_ARG;
    K4_CUDA_TRY(cudaFuncSetAttribute(png_match_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)MATCH_SMEM));
    K4_CUDA_TRY(cudaFuncSetAttribute(png_encode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ENC_SMEM));
    const cudaStream_t st = (cudaStream_t)stream;
    const int64_t n = png_n(H, W), nseg = png_nseg(n);
    const PngWs L = png_ws_layout(H, W);
    uint8_t* ws = (uint8_t*)d_workspace;
    uint8_t* filt = ws + L.filt;
    uint32_t* best = (uint32_t*)(ws + L.best);
    uint8_t* segout = ws + L.segout;
    uint32_t* seglen = (uint32_t*)(ws + L.seglen);
    int64_t* segoff = (int64_t*)(ws + L.segoff);
    uint32_t* segadl = (uint32_t*)(ws + L.segadl);
    uint32_t* crc = (uint32_t*)(ws + L.crc);
    int64_t* misc = (int64_t*)(ws + L.misc);

    PngHead head;
    const uint8_t sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1a, '\n'};
    for (int i = 0; i < 8; ++i) head.b[i] = sig[i];
    uint8_t* ih = head.b + 8;
    const uint8_t ihdr[25] = {0, 0, 0, 13, 'I', 'H', 'D', 'R',
                              (uint8_t)(W >> 24), (uint8_t)(W >> 16), (uint8_t)(W >> 8), (uint8_t)W,
                              (uint8_t)(H >> 24), (uint8_t)(H >> 16), (uint8_t)(H >> 8), (uint8_t)H,
                              8, 2, 0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < 25; ++i) ih[i] = ihdr[i];
    uint32_t c = 0xffffffffu;
    for (int i = 4; i < 21; ++i) c = crc_byte_update(c, ih[i]);
    c ^= 0xffffffffu;
    ih[21] = (uint8_t)(c >> 24); ih[22] = (uint8_t)(c >> 16); ih[23] = (uint8_t)(c >> 8); ih[24] = (uint8_t)c;

    png_filter_kernel<<<(unsigned)((H + 7) / 8), 256, 0, st>>>(d_rgb, (int)H, (int)W, filt);
    png_match_kernel<<<(unsigned)nseg, NT, MATCH_SMEM, st>>>(filt, n, (int)min((int64_t)1 << 30, 1 + 3 * W), best);
    png_encode_kernel<<<(unsigned)nseg, NT, ENC_SMEM, st>>>(filt, n, best, segout, seglen, segadl);
    png_join_kernel<<<1, NT, 0, st>>>(seglen, segadl, n, nseg, segoff, misc, head, d_out, d_len);
    png_copy_kernel<<<(unsigned)nseg, 256, 0, st>>>(segout, seglen, segoff, d_out);
    const int64_t npieces = (int64_t)((k4_png_encode_bound(H, W) - HDR - 10) / CRC_PIECE) + 1;
    png_crc_kernel<<<(unsigned)((npieces + 255) / 256), 256, 0, st>>>(d_out, misc, npieces, crc);
    png_crc_join_kernel<<<1, NT, 0, st>>>(crc, misc, d_out);
    return launch_error("k4_png_encode launch");
}

int k4_testing_png_code_lengths(const int32_t* d_freq, int32_t n, int32_t maxbits, uint8_t* d_len, k4_stream_t stream) {
    if (!d_freq || !d_len || n < 1 || n > MAXSYM || maxbits < 1 || maxbits > 15) return K4_ERR_INVALID_ARG;
    png_code_lengths_kernel<<<1, NT, 0, (cudaStream_t)stream>>>(d_freq, n, maxbits, d_len);
    return launch_error("k4_testing_png_code_lengths launch");
}

}  // extern "C"
