/*
 * regk_core.cuh — per-record composers of the registration hot path, written
 * as word-at-a-time (SWAR) byte manipulation so that one GPU thread can turn
 * one service record into its znode path and its JSON payload with a few
 * hundred integer instructions and 32-bit shared-memory accesses.
 *
 * Reference semantics restated here (relative to /root/reference):
 *   A1  lib/register.js:34-39   domainToPath(): lower-case, split on '.',
 *                               reverse, join with '/', leading '/'
 *   A2  lib/register.js:221-223 path.join(p, os.hostname()): posix normalise
 *                               (empty labels vanish), '/' + hostname appended
 *   A3  lib/register.js:141-155 host-record object, key order type, address,
 *                               ttl, <type>:{address, ports}
 *   A4  lib/register.js:159     zkplus JSON.stringify -> compact JSON bytes
 *
 * Everything is templated on a word source (where the record's input bytes
 * live) and a byte sink (where output bytes go) so the same code serves the
 * shared-memory fast path, the direct-to-global generic path, and the CPU
 * logic tests in tests/ (RG_HD expands to nothing under a host compiler).
 */
#ifndef REGK_CORE_CUH
#define REGK_CORE_CUH

#include <stddef.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define RG_HD __host__ __device__ __forceinline__
#define RG_D __device__ __forceinline__
#else
#define RG_HD inline
#define RG_D inline
#endif

namespace regk {

/* 16-byte vector: one LDS.128 / STS.128 per thread on the GPU (consecutive threads -> conflict-free) */
#if defined(__CUDACC__)
typedef uint4 Quad;
#else
struct alignas(16) Quad {
    uint32_t x, y, z, w;
};
#endif

/* validation bits: keep in sync with include/regk.h */
enum : uint32_t {
    BAD_DOMAIN_BYTE = 1u << 0,
    BAD_HOST_BYTE = 1u << 1,
    BAD_ADDR_BYTE = 1u << 2,
    BAD_TYPE_ID = 1u << 3,
    BAD_TOO_LARGE = 1u << 4,
    BAD_SERVICE_BYTE = 1u << 5,
    BAD_KEY_ORDER = 1u << 6,
};

/* ---------------------------------------------------------------- SWAR -- */

RG_HD uint32_t funnel_r(uint32_t lo, uint32_t hi, uint32_t shift_bits)
{
#if defined(__CUDA_ARCH__)
    return __funnelshift_r(lo, hi, shift_bits);          /* shift_bits in [0, 31] */
#else
    return (uint32_t)(((((uint64_t)hi) << 32) | lo) >> (shift_bits & 31));
#endif
}

/* left funnel shift: the high word of (hi:lo) << shift_bits, shift_bits in [0, 31] */
RG_HD uint32_t funnel_l(uint32_t lo, uint32_t hi, uint32_t shift_bits)
{
#if defined(__CUDA_ARCH__)
    return __funnelshift_l(lo, hi, shift_bits);
#else
    return (uint32_t)((((((uint64_t)hi) << 32) | lo) << (shift_bits & 31)) >> 32);
#endif
}

/* right funnel shift with the shift amount clamped to 32 (shift == 32 returns hi) */
RG_HD uint32_t funnel_rc(uint32_t lo, uint32_t hi, uint32_t shift_bits)
{
#if defined(__CUDA_ARCH__)
    return __funnelshift_rc(lo, hi, shift_bits);
#else
    return shift_bits >= 32 ? hi : (uint32_t)(((((uint64_t)hi) << 32) | lo) >> shift_bits);
#endif
}

RG_HD uint32_t popc64(uint64_t v)
{
#if defined(__CUDA_ARCH__)
    return (uint32_t)__popcll(v);
#else
    return (uint32_t)__builtin_popcountll(v);
#endif
}

RG_HD uint32_t clz64(uint64_t v)
{
#if defined(__CUDA_ARCH__)
    return (uint32_t)__clzll((long long)v);
#else
    return v ? (uint32_t)__builtin_clzll(v) : 64u;
#endif
}

RG_HD uint32_t popc32(uint32_t v)
{
#if defined(__CUDA_ARCH__)
    return (uint32_t)__popc(v);
#else
    return (uint32_t)__builtin_popcount(v);
#endif
}

RG_HD uint32_t clz32(uint32_t v)
{
#if defined(__CUDA_ARCH__)
    return (uint32_t)__clz((int)v);
#else
    return v ? (uint32_t)__builtin_clz(v) : 32u;
#endif
}

/* mask with the low n bytes set, n in [0, 4] */
RG_HD uint32_t low_bytes(uint32_t n)
{
    return n >= 4 ? 0xFFFFFFFFu : ((1u << (8 * n)) - 1u);
}

/* For a word of 7-bit bytes: bit 7 of every byte that equals c (exact per byte). */
RG_HD uint32_t eq7(uint32_t v7, uint32_t c)
{
    uint32_t x = v7 ^ (c * 0x01010101u);                 /* 0 where equal, still 7-bit */
    return ~(x + 0x7F7F7F7Fu) & 0x80808080u;             /* no inter-byte carry for 7-bit bytes */
}

/* For a word of 7-bit bytes: bit 7 of every byte that is zero after masking with m. */
RG_HD uint32_t zero7(uint32_t v7)
{
    return ~(v7 + 0x7F7F7F7Fu) & 0x80808080u;
}

/* ASCII lower-casing of 4 bytes (7-bit bytes): 'A'..'Z' -> 'a'..'z'  (String.prototype.toLowerCase
 * restricted to ASCII, lib/register.js:38). */
RG_HD uint32_t lower7(uint32_t v7)
{
    uint32_t ge_A = v7 + 0x3F3F3F3Fu;                    /* bit7 iff byte >= 0x41 */
    uint32_t gt_Z = v7 + 0x25252525u;                    /* bit7 iff byte >= 0x5B */
    uint32_t up = ge_A & ~gt_Z & 0x80808080u;
    return v7 | (up >> 2);                               /* + 0x20 */
}

/* ---------------------------------------------------------------- sinks -- */

/*
 * WordSink: sequential byte writer into a 32-bit-word image of the tile's output
 * (shared memory on the GPU).  Pending bytes live in a 32-bit carry; a word is
 * stored the moment its last byte is known, so exactly one thread — the owner of
 * the word's last byte — ever stores a given word.  Words shared by neighbouring
 * records are resolved in two phases separated by a block barrier:
 *   phase A  (put / put4):  full-word stores; the low bytes of a record's first word
 *            that belong to the previous record are stored as zero;
 *   phase B  (tail):        every record writes its last, incomplete word byte by
 *            byte (at most 3 bytes), filling those zeros in.
 * There is no per-store branch on "is this the first word".
 */
struct WordSink {
    uint32_t *wp;           /* the word being filled */
    uint32_t carry;         /* its bytes so far (low `s` bits) */
    uint32_t s;             /* pending bits: 0, 8, 16 or 24 */
    uint32_t *wp0;          /* first word of the record ... */
    uint32_t h0;            /* ... and the number of foreign bytes in it */

    RG_HD void init(uint32_t *base, uint32_t byte_off)
    {
        wp = wp0 = base + (byte_off >> 2);
        h0 = byte_off & 3u;
        s = h0 * 8u;
        carry = 0;
    }
    RG_HD void put4(uint32_t v)
    {
        *wp++ = carry | (v << s);
        carry = funnel_rc(v, 0u, 32u - s);
    }
    /* N whole words in a row: one funnel shift per word instead of shift + or + carry */
    template <int N>
    RG_HD void put_words(const uint32_t (&v)[N])
    {
        wp[0] = carry | (v[0] << s);
        #pragma unroll
        for (int i = 1; i < N; i++)
            wp[i] = funnel_l(v[i - 1], v[i], s);
        carry = funnel_rc(v[N - 1], 0u, 32u - s);
        wp += N;
    }
    /* append the low n bytes of v (1 <= n <= 4); bytes of v above n must be zero */
    RG_HD void put(uint32_t v, uint32_t n)
    {
        const uint32_t out = carry | (v << s);
        const uint32_t ns = s + 8u * n;
        const bool full = ns >= 32u;
        if (full)
            *wp = out;
        wp += full ? 1 : 0;
        carry = full ? funnel_rc(v, 0u, 32u - s) : out;
        s = full ? ns - 32u : ns;
    }
    /* append the low n bytes (1..8) of the 64-bit little-endian value hi:lo; bytes above n must be zero */
    RG_HD void put8(uint32_t lo, uint32_t hi, uint32_t n)
    {
        const uint32_t back = 32u - s;
        const uint32_t o0 = carry | (lo << s);
        const uint32_t o1 = funnel_rc(lo, hi, back);
        const uint32_t o2 = funnel_rc(hi, 0u, back);
        const uint32_t total = (s >> 3) + n;                /* 1..11 bytes pending */
        if (total >= 4u)
            wp[0] = o0;
        if (total >= 8u)
            wp[1] = o1;
        const uint32_t nf = total >> 2;                     /* completed words: 0..2 */
        carry = nf == 0u ? o0 : nf == 1u ? o1 : o2;
        wp += nf;
        s = (total & 3u) * 8u;
    }
    RG_HD void put1(uint32_t c)
    {
        const uint32_t out = carry | (c << s);
        const bool full = s == 24u;
        if (full)
            *wp = out;
        wp += full ? 1 : 0;
        carry = full ? 0u : out;
        s = full ? 0u : s + 8u;
    }
    RG_HD void finish() {}
    /* phase B: after every thread of the tile has finished phase A */
    RG_HD void tail()
    {
        uint8_t *b = reinterpret_cast<uint8_t *>(wp);
        const uint32_t lo = (wp == wp0) ? h0 : 0u;
        const uint32_t hi = s >> 3;
        if (lo <= 0u && hi > 0u)
            b[0] = (uint8_t)carry;
        if (lo <= 1u && hi > 1u)
            b[1] = (uint8_t)(carry >> 8);
        if (lo <= 2u && hi > 2u)
            b[2] = (uint8_t)(carry >> 16);
    }
};

/* ByteSink: same interface, writes straight to a byte pointer (generic path / CPU tests). */
struct ByteSink {
    uint8_t *p;
    RG_HD void init(uint8_t *dst) { p = dst; }
    RG_HD void put(uint32_t v, uint32_t n)
    {
        for (uint32_t k = 0; k < n; k++)
            *p++ = (uint8_t)(v >> (8 * k));
    }
    RG_HD void put4(uint32_t v) { put(v, 4); }
    RG_HD void put8(uint32_t lo, uint32_t hi, uint32_t n)
    {
        put(lo, n < 4u ? n : 4u);
        if (n > 4u)
            put(hi, n - 4u);
    }
    RG_HD void put1(uint32_t c) { *p++ = (uint8_t)c; }
    RG_HD void finish() {}
    RG_HD void tail() {}
};

/* CountSink: length only. */
struct CountSink {
    uint32_t n;
    RG_HD void init() { n = 0; }
    RG_HD void put(uint32_t, uint32_t k) { n += k; }
    RG_HD void put4(uint32_t) { n += 4; }
    RG_HD void put8(uint32_t, uint32_t, uint32_t k) { n += k; }
    RG_HD void put1(uint32_t) { n += 1; }
    RG_HD void finish() {}
};

/* -------------------------------------------------------------- sources -- */

/* Word source over an aligned 32-bit buffer that is readable one word past the
 * last byte used (shared-memory staging buffers are padded accordingly). */
struct PaddedWords {
    const uint32_t *w;
    RG_HD uint32_t word(uint32_t i) const { return w[i]; }
    RG_HD uint32_t word_hi(uint32_t i, uint32_t /*needed*/) const { return w[i]; }
};

/* Word source over global memory: never touches a word that holds no needed byte. */
struct GuardedWords {
    const uint32_t *w;
    RG_HD uint32_t word(uint32_t i) const { return w[i]; }
    RG_HD uint32_t word_hi(uint32_t i, uint32_t needed) const { return needed ? w[i] : 0u; }
};

/*
 * Copy len bytes starting at byte offset `off` of `src` into `sink`, optionally
 * lower-casing, and OR the raw bytes into *seen (for validation).  One source
 * word load and one sink word per 4 bytes.
 */
template <bool LOWER, class Src, class Sink>
RG_HD void copy_bytes(const Src &src, uint32_t off, uint32_t len, Sink &sink)
{
    if (len == 0)
        return;
    uint32_t wi = off >> 2;
    const uint32_t sh = (off & 3u) * 8u;
    uint32_t lo = src.word(wi);
    while (len >= 4) {
        /* the next word is needed iff the 4 bytes straddle it */
        uint32_t hi = src.word_hi(wi + 1, sh != 0 || len > 4);
        uint32_t v = funnel_r(lo, hi, sh);
        if (LOWER)
            v = lower7(v & 0x7F7F7F7Fu);
        sink.put4(v);
        lo = hi;
        wi++;
        len -= 4;
    }
    if (len) {
        uint32_t hi = src.word_hi(wi + 1, sh + 8 * len > 32);
        uint32_t v = funnel_r(lo, hi, sh) & low_bytes(len);
        if (LOWER)
            v = lower7(v & 0x7F7F7F7Fu);
        sink.put(v, len);
    }
}

/* ------------------------------------------------------ A1/A2: the path -- */

struct DomainStats {
    uint32_t nondot;        /* bytes that are not '.' */
    uint32_t labels;        /* non-empty labels */
    uint32_t bad;           /* REGK_BAD_DOMAIN_BYTE or 0 */
};

/*
 * One forward pass over the domain (bytes [off, off+L) of src): counts what the
 * path length needs and applies the input fence (byte >= 0x80 or '/').
 */
template <class Src>
RG_HD DomainStats scan_domain(const Src &src, uint32_t off, uint32_t L)
{
    DomainStats st;
    st.nondot = 0;
    st.labels = 0;
    st.bad = 0;
    if (L == 0)
        return st;
    uint32_t wi = off >> 2;
    const uint32_t sh = (off & 3u) * 8u;
    uint32_t lo = src.word(wi);
    uint32_t prev_dot = 0x80u;          /* position -1 counts as a separator */
    uint32_t hibits = 0, slash = 0;
    uint32_t rem = L;
    while (rem) {
        uint32_t nbytes = rem < 4 ? rem : 4;
        uint32_t hi = src.word_hi(wi + 1, sh + 8 * nbytes > 32 || rem > 4);
        uint32_t v = funnel_r(lo, hi, sh);
        uint32_t keep = low_bytes(nbytes);
        v &= keep;
        hibits |= v;
        uint32_t v7 = v & 0x7F7F7F7Fu;
        uint32_t x = v7 ^ 0x2E2E2E2Eu;                      /* '.' -> 0x00, '/' -> 0x01 */
        uint32_t dot = zero7(x);
        uint32_t dot_or_slash = zero7(x & 0x7E7E7E7Eu);
        slash |= (dot ^ dot_or_slash) & (keep & 0x80808080u);
        uint32_t valid7 = keep & 0x80808080u;
        uint32_t nd = ~dot & valid7;                        /* non-dot bytes inside the domain */
        uint32_t before = (dot << 8) | prev_dot;            /* bit7 of byte k set iff byte k-1 is a separator */
        st.nondot += popc32(nd);
        st.labels += popc32(nd & before);
        prev_dot = dot >> 24;
        lo = hi;
        wi++;
        rem -= nbytes;
    }
    if ((hibits & 0x80808080u) || slash)
        st.bad = BAD_DOMAIN_BYTE;
    return st;
}

/* Absolute byte position of the last '.' in [a, e) of src, or a - 1 when there is none (e > a). */
template <class Src>
RG_HD int32_t find_prev_dot(const Src &src, uint32_t a, uint32_t e)
{
    uint32_t wi = (e - 1) >> 2;
    uint32_t nkeep = e - 4 * wi;                            /* 1..4 bytes of this word are below e */
    uint32_t dm = eq7(src.word(wi) & 0x7F7F7F7Fu, 0x2E) & low_bytes(nkeep);
    for (;;) {
        if (dm) {
            int32_t pos = (int32_t)(4 * wi + ((31u - clz32(dm)) >> 3));
            return pos >= (int32_t)a ? pos : (int32_t)a - 1;
        }
        if (4 * wi <= a)
            return (int32_t)a - 1;
        wi--;
        dm = eq7(src.word(wi) & 0x7F7F7F7Fu, 0x2E);
    }
}

/*
 * Emit the znode path of one record.
 *   ALIAS = false: host node, path.join(domainToPath(domain), hostname) (A2):
 *                  '/' + each non-empty label from last to first + '/' ... + '/' + hostname
 *   ALIAS = true : alias node, domainToPath(domain) un-normalised (A1): every label,
 *                  empty ones included, preceded by '/'
 * dom: bytes [doff, doff+L) of dsrc; host: bytes [hoff, hoff+H) of hsrc.
 */
template <bool ALIAS, class DSrc, class HSrc, class Sink>
RG_HD void emit_path(const DSrc &dsrc, uint32_t doff, uint32_t L, const HSrc &hsrc, uint32_t hoff,
    uint32_t H, Sink &sink)
{
    uint32_t e = doff + L;                                  /* end (exclusive) of the current label */
    for (;;) {
        int32_t dot = e > doff ? find_prev_dot(dsrc, doff, e) : (int32_t)doff - 1;
        uint32_t s = (uint32_t)(dot + 1);
        if (ALIAS || e > s) {
            sink.put1('/');
            copy_bytes<true>(dsrc, s, e - s, sink);
        }
        if (s == doff)
            break;
        e = s - 1;
    }
    if (!ALIAS) {
        sink.put1('/');
        copy_bytes<false>(hsrc, hoff, H, sink);
    }
}

RG_HD uint32_t path_length(const DomainStats &st, uint32_t L, uint32_t H, bool alias)
{
    return alias ? L + 1 : 1 + st.nondot + st.labels + H;
}

/* Hostname fence: non-empty, not "." / "..", bytes in 0x01..0x7f except '/'. */
template <class Src>
RG_HD uint32_t check_host(const Src &src, uint32_t off, uint32_t H)
{
    if (H == 0)
        return BAD_HOST_BYTE;
    uint32_t wi = off >> 2;
    const uint32_t sh = (off & 3u) * 8u;
    uint32_t lo = src.word(wi);
    uint32_t hibits = 0, hit = 0, first = 0;
    uint32_t rem = H;
    bool is_first = true;
    while (rem) {
        uint32_t nbytes = rem < 4 ? rem : 4;
        uint32_t hi = src.word_hi(wi + 1, sh + 8 * nbytes > 32 || rem > 4);
        uint32_t keep = low_bytes(nbytes);
        uint32_t v = funnel_r(lo, hi, sh) & keep;
        if (is_first) {
            first = v;
            is_first = false;
        }
        hibits |= v;
        uint32_t v7 = v & 0x7F7F7F7Fu;
        hit |= (eq7(v7, 0x2F) | zero7(v7)) & keep;          /* '/' or NUL */
        lo = hi;
        wi++;
        rem -= nbytes;
    }
    bool dots = (H == 1 && first == 0x2Eu) || (H == 2 && first == 0x2E2Eu);
    return ((hibits & 0x80808080u) || hit || dots) ? (uint32_t)BAD_HOST_BYTE : 0u;
}

/* ------------------------------------------- tile-cooperative pre-pass -- */

/* bits 7/15/23/31 of m -> bits 0..3 */
RG_HD uint32_t movemask4(uint32_t m)
{
    return (((m >> 7) * 0x00204081u) >> 21) & 0xFu;
}

/*
 * Domain pre-pass over the staged bytes of a tile, 16 bytes per step, thread t of
 * nt takes chunks t, t+nt, ...: lower-cases ASCII letters in place (A1,
 * toLowerCase), records one "is '.'" bit per byte in `bits` (16 bits per chunk),
 * rewrites every '.' to '/' in place (so a label can be copied together with the
 * separator in front of it) and returns nonzero if a byte outside the fence
 * (>= 0x80 or '/') was seen anywhere in the chunks it handled — the caller then
 * re-validates record by record (recheck_domain).
 */
RG_HD uint32_t prepass_domain(uint32_t *dom_words, uint16_t *bits, uint32_t nchunks, uint32_t t, uint32_t nt)
{
    uint32_t hib = 0, slash = 0;
    Quad *q = reinterpret_cast<Quad *>(dom_words);
    for (uint32_t c = t; c < nchunks; c += nt) {
        const Quad in = q[c];                               /* one 128-bit shared-memory access per thread */
        uint32_t wv[4] = {in.x, in.y, in.z, in.w};
        uint32_t m = 0;
        #pragma unroll
        for (int j = 0; j < 4; j++) {
            const uint32_t w = wv[j];
            const uint32_t v7 = w & 0x7F7F7F7Fu;
            const uint32_t x = v7 ^ 0x2E2E2E2Eu;                /* '.' -> 0x00, '/' -> 0x01 */
            const uint32_t dot = zero7(x);
            slash |= dot ^ zero7(x & 0x7E7E7E7Eu);
            hib |= w;
            wv[j] = lower7(v7) | (w & 0x80808080u) | (dot >> 7);    /* 0x2e | 1 = 0x2f */
            m |= movemask4(dot) << (4 * j);
        }
        Quad out;
        out.x = wv[0];
        out.y = wv[1];
        out.z = wv[2];
        out.w = wv[3];
        q[c] = out;
        bits[c] = (uint16_t)m;
    }
    return (hib & 0x80808080u) | slash;
}

/* Hostname pre-pass: nonzero if any staged byte is >= 0x80, NUL or '/'.  Uses the borrow-based "has a zero
 * byte" test ((v - 0x01..) & ~v & 0x80..), which is exact as a yes/no answer over the word. */
RG_HD uint32_t prepass_host(const uint32_t *host_words, uint32_t nchunks, uint32_t t, uint32_t nt)
{
    uint32_t acc = 0;
    const Quad *q = reinterpret_cast<const Quad *>(host_words);
    for (uint32_t c = t; c < nchunks; c += nt) {
        const Quad in = q[c];                               /* one 128-bit shared-memory access per thread */
        const uint32_t wv[4] = {in.x, in.y, in.z, in.w};
        #pragma unroll
        for (int j = 0; j < 4; j++) {
            const uint32_t w = wv[j];
            const uint32_t x = w ^ 0x2F2F2F2Fu;
            acc |= w | ((w - 0x01010101u) & ~w) | ((x - 0x01010101u) & ~x);
        }
    }
    return acc & 0x80808080u;
}

/* exact per-record domain fence on pre-passed bytes (dots already rewritten to '/'): rare path */
RG_HD uint32_t recheck_domain(const uint8_t *dom, const uint32_t *bits, uint32_t doff, uint32_t L)
{
    for (uint32_t i = 0; i < L; i++) {
        const uint32_t c = dom[doff + i], b = doff + i;
        const bool is_dot = (bits[b >> 5] >> (b & 31u)) & 1u;
        if (c >= 0x80u || (c == 0x2Fu && !is_dot))
            return BAD_DOMAIN_BYTE;
    }
    return 0;
}

/* What the path needs to know about one domain, from the dot bitmap. */
struct DomainInfo {
    uint64_t dots;          /* bit i = byte i is '.', valid when small */
    uint32_t nondot;
    uint32_t labels;        /* non-empty labels */
    bool small;             /* L <= 64: `dots` describes the whole domain */
};

RG_HD uint32_t bit_window32(const uint32_t *bits, uint32_t pos)
{
    return funnel_r(bits[pos >> 5], bits[(pos >> 5) + 1], pos & 31u);
}

/* 64 bitmap bits starting at bit `pos` (the bitmap is readable two words past its end) */
RG_HD uint64_t bit_window64(const uint32_t *bits, uint32_t pos)
{
    const uint32_t wi = pos >> 5, sh = pos & 31u;
    const uint32_t w0 = bits[wi], w1 = bits[wi + 1], w2 = bits[wi + 2];
    return ((uint64_t)funnel_r(w1, w2, sh) << 32) | funnel_r(w0, w1, sh);
}

/* bits: dot bitmap of the staged tile (readable two words past the end); b0: bit index of the domain's byte 0 */
RG_HD DomainInfo domain_info(const uint32_t *bits, uint32_t b0, uint32_t L)
{
    DomainInfo di;
    di.small = L <= 64u;
    if (di.small) {
        const uint32_t wi = b0 >> 5, sh = b0 & 31u;
        const uint32_t w0 = bits[wi], w1 = bits[wi + 1], w2 = bits[wi + 2];
        const uint64_t win = ((uint64_t)funnel_r(w1, w2, sh) << 32) | funnel_r(w0, w1, sh);
        const uint64_t mask = L >= 64u ? ~0ull : ((1ull << L) - 1ull);
        di.dots = win & mask;
        const uint64_t nd = ~di.dots & mask;
        di.nondot = popc64(nd);
        di.labels = popc64(nd & ((di.dots << 1) | 1ull));
    } else {
        di.dots = 0;
        di.nondot = 0;
        di.labels = 0;
        uint32_t carry = 1u, pos = b0, rem = L;
        while (rem) {
            const uint32_t n = rem < 32u ? rem : 32u;
            const uint32_t mask = n >= 32u ? 0xFFFFFFFFu : ((1u << n) - 1u);
            const uint32_t w = bit_window32(bits, pos) & mask;
            const uint32_t nd = ~w & mask;
            di.nondot += popc32(nd);
            di.labels += popc32(nd & ((w << 1) | carry));
            carry = (w >> (n - 1u)) & 1u;
            pos += n;
            rem -= n;
        }
    }
    return di;
}

RG_HD uint32_t path_length2(const DomainInfo &di, uint32_t L, uint32_t H, bool alias)
{
    return alias ? L + 1u : 1u + di.nondot + di.labels + H;
}

/* 16 bytes starting at byte offset `off` of a padded word buffer -> 4 registers (5 loads, 4 funnel shifts) */
RG_HD void load16(const uint32_t *w, uint32_t off, uint32_t (&a)[4])
{
    const uint32_t *p = w + (off >> 2);
    const uint32_t sh = (off & 3u) * 8u;
    const uint32_t w0 = p[0], w1 = p[1], w2 = p[2], w3 = p[3], w4 = p[4];
    a[0] = funnel_r(w0, w1, sh);
    a[1] = funnel_r(w1, w2, sh);
    a[2] = funnel_r(w2, w3, sh);
    a[3] = funnel_r(w3, w4, sh);
}

/*
 * Append the first n (1..16) bytes of a 16-byte register block; bytes of a[] beyond n may be anything.
 *
 * OVERSHOOT = true: straight-line code — the five candidate words are all stored and the new carry is read
 * back from the word that stays open.  Up to 20 bytes past the sink's current word are overwritten with
 * garbage, so it may only be used while at least 24 more bytes of the SAME record follow (they are written
 * later by this thread, and the record's last, possibly shared, word is never touched).
 * OVERSHOOT = false: exact stores, for the end of a record.
 */
template <bool OVERSHOOT>
RG_HD void put_block16(const uint32_t (&a)[4], uint32_t n, WordSink &sink)
{
    const uint32_t sh = sink.s, back = 32u - sh;
    const uint32_t o0 = sink.carry | (a[0] << sh);
    const uint32_t o1 = funnel_rc(a[0], a[1], back);
    const uint32_t o2 = funnel_rc(a[1], a[2], back);
    const uint32_t o3 = funnel_rc(a[2], a[3], back);
    const uint32_t o4 = funnel_rc(a[3], 0u, back);
    const uint32_t total = (sh >> 3) + n;
    const uint32_t nfull = total >> 2, rem = total & 3u;
    uint32_t *dst = sink.wp;
    uint32_t c;
    if (OVERSHOOT) {
        dst[0] = o0;
        dst[1] = o1;
        dst[2] = o2;
        dst[3] = o3;
        dst[4] = o4;
        c = dst[nfull];
    } else {
        if (nfull > 0) dst[0] = o0;
        if (nfull > 1) dst[1] = o1;
        if (nfull > 2) dst[2] = o2;
        if (nfull > 3) dst[3] = o3;
        c = nfull == 0 ? o0 : nfull == 1 ? o1 : nfull == 2 ? o2 : nfull == 3 ? o3 : o4;
    }
    sink.carry = c & low_bytes(rem);
    sink.wp = dst + nfull;
    sink.s = rem * 8u;
}

/* copy len bytes from a padded word buffer in 16-byte register blocks */
template <bool OVERSHOOT>
RG_HD void copy_blocks(const uint32_t *w, uint32_t off, uint32_t len, WordSink &sink)
{
    uint32_t a[4];
    while (len) {
        const uint32_t n = len < 16u ? len : 16u;
        load16(w, off, a);
        put_block16<OVERSHOOT>(a, n, sink);
        off += 16u;
        len -= n;
    }
}

/*
 * Emit one znode path from pre-passed shared-memory inputs (see emit_path for the semantics).
 * `dom` holds lower-cased bytes with every '.' already rewritten to '/', and is readable from 16 bytes
 * BEFORE its nominal start (`doff` is relative to dom, the caller passes dom = staged buffer + 16 bytes).
 * Every label is copied together with the byte in front of it — the separator, already a '/'; for the
 * label at offset 0 that byte belongs to someone else and is patched to '/' in the register block — so the
 * label loop has no special cases.  Label boundaries come from the dot bitmap: the highest remaining dot of a
 * 64-bit window is one clz away and is cleared after use; domains longer than 64 bytes slide the window down.
 * FAST: a hostname of >= 24 bytes follows the labels, so label blocks may overshoot (put_block16).
 */
template <bool ALIAS, bool FAST>
RG_HD void emit_path2(const uint32_t *dom, const uint32_t *bits, uint32_t doff, uint32_t L, const DomainInfo &di,
    const uint32_t *host, uint32_t hoff, uint32_t H, WordSink &sink)
{
    /* Labels are found from the end with one clz per label in a 64-bit window of the dot bitmap, bit i of the
       window = domain byte wbase + i.  Domains of up to 64 bytes have the whole bitmap in the window (wbase = 0);
       longer ones start at their last 64 bytes and slide the window down when it runs out of dots. */
    uint32_t e = L;                                         /* end (exclusive) of the current label, relative */
    uint32_t wbase = di.small ? 0u : L - 64u;
    uint64_t dots = di.small ? di.dots : bit_window64(bits, doff + wbase);
    for (;;) {
        while (dots == 0 && wbase != 0) {                   /* nothing left in this window: look further down */
            const uint32_t nb = wbase < 64u ? wbase : 64u;
            wbase -= nb;
            const uint64_t w = bit_window64(bits, doff + wbase);
            dots = nb >= 64u ? w : (w & ((1ull << nb) - 1ull));     /* only positions below the old window */
        }
        const uint32_t s = dots ? wbase + 64u - clz64(dots) : 0u;   /* position after the highest remaining '.', or 0 */
        if (ALIAS || e > s) {
            /* bytes [s-1, e): separator + label, in 16-byte register blocks */
            uint32_t off = doff + s - 1u, len = e - s + 1u;
            uint32_t a[4];
            load16(dom - 4, off + 16u, a);                  /* dom - 4 words = 16 bytes of front padding */
            if (s == 0)
                a[0] = (a[0] & 0xFFFFFF00u) | 0x2Fu;
            for (;;) {
                const uint32_t n = len < 16u ? len : 16u;
                put_block16<FAST>(a, n, sink);
                len -= n;
                if (len == 0)
                    break;
                off += 16u;
                load16(dom - 4, off + 16u, a);
            }
        }
        if (s == 0)
            break;
        dots &= ~(1ull << (s - 1u - wbase));
        e = s - 1u;
    }
    if (!ALIAS) {
        sink.put1('/');
        if (((hoff | H) & 3u) == 0) {
            const uint32_t *hw = host + (hoff >> 2);
            const uint32_t nw = H >> 2;
            if (nw == 9) {                                  /* 36-byte UUID: all loads in flight, then the stores */
                uint32_t h[9];
                #pragma unroll
                for (int i = 0; i < 9; i++)
                    h[i] = hw[i];
                sink.put_words(h);
            } else {
                for (uint32_t i = 0; i < nw; i++)
                    sink.put4(hw[i]);
            }
        } else {
            copy_blocks<false>(host, hoff, H, sink);
        }
    }
}

/* --------------------------------------------------- A3/A4: the payload -- */

/* Decimal digits of r < 10000 as 4 ASCII bytes, most significant digit in byte 0. */
RG_HD uint32_t dec4(uint32_t r)
{
    uint32_t hi = (r * 5243u) >> 19;                        /* r / 100 for r < 10000 */
    uint32_t lo = r - hi * 100u;
    uint32_t pair = hi | (lo << 16);                        /* two values < 100 in 16-bit lanes */
    uint32_t tens = ((pair * 103u) >> 10) & 0x000F000Fu;    /* x / 10 for x < 100, per lane */
    uint32_t ones = pair - tens * 10u;
    return (tens | (ones << 8)) + 0x30303030u;
}

RG_HD uint32_t ndigits4(uint32_t r)                          /* r < 10000 */
{
    return 1u + (r >= 10u) + (r >= 100u) + (r >= 1000u);
}

/* decimal digits of any uint32, branch-free: floor(log10) estimated from the bit length (1233/4096 ~ log10 2),
   corrected by one table compare.  (v | 1 keeps 0 at one digit; 10^t - 1 is odd, so the `| 1` changes no answer.) */
#if defined(__CUDACC__)
__device__ __constant__ uint32_t regk_pow10_dev[10] = {1u, 10u, 100u, 1000u, 10000u, 100000u, 1000000u, 10000000u,
                                                       100000000u, 1000000000u};
#endif
RG_HD uint32_t pow10_u32(uint32_t t)                        /* t in 0..9 */
{
#if defined(__CUDA_ARCH__)
    return regk_pow10_dev[t];                               /* constant bank, not a stack array */
#else
    static const uint32_t p10[10] = {1u, 10u, 100u, 1000u, 10000u, 100000u, 1000000u, 10000000u, 100000000u, 1000000000u};
    return p10[t];
#endif
}

RG_HD uint32_t ndigits_u32(uint32_t v)
{
    const uint32_t w = v | 1u;
    const uint32_t t = ((32u - clz32(w)) * 1233u) >> 12;    /* 0..9 */
    return t + 1u - (w < pow10_u32(t) ? 1u : 0u);
}

/* Number::toString for an unsigned 32-bit integer (ports, |ttl|). */
template <class Sink>
RG_HD void put_u32_dec(uint32_t v, Sink &sink)
{
    if (v < 10000u) {
        uint32_t n = ndigits4(v);
        sink.put(dec4(v) >> (8 * (4 - n)), n);
        return;
    }
    uint32_t q = v / 10000u, r = v - q * 10000u;
    if (q < 10000u) {
        uint32_t n = ndigits4(q);
        sink.put(dec4(q) >> (8 * (4 - n)), n);
    } else {
        uint32_t q2 = q / 10000u, r2 = q - q2 * 10000u;     /* q2 <= 42 */
        uint32_t n = ndigits4(q2);
        sink.put(dec4(q2) >> (8 * (4 - n)), n);
        sink.put4(dec4(r2));
    }
    sink.put4(dec4(r));
}

/* One element of "ports":[...] with the comma in front of it (not for the first): values below 100000 - every
   TCP/UDP port - are composed in registers (comma, leading digit, four SWAR digits) and appended by ONE sink
   operation; anything larger takes the general integer path. */
template <class Sink>
RG_HD void put_port(uint32_t v, bool comma, Sink &sink)
{
    if (v >= 100000u) {
        if (comma)
            sink.put1(',');
        put_u32_dec(v, sink);
        return;
    }
    const uint32_t q = v / 10000u;                          /* 0..9 (a multiply-high and a shift) */
    const uint32_t r = v - q * 10000u;
    const uint32_t d4 = dec4(r);                            /* four ASCII digits, most significant in byte 0 */
    const uint32_t n4 = q ? 4u : ndigits4(r);
    uint32_t lo = d4 >> (8u * (4u - n4)), hi = 0, n = n4;   /* the low-order digits, leading zeros dropped */
    if (q) {                                                /* five digits: the leading one goes in front */
        hi = lo >> 24;
        lo = (lo << 8) | (q + 0x30u);
        n = 5u;
    }
    if (comma) {
        hi = (hi << 8) | (lo >> 24);
        lo = (lo << 8) | 0x2Cu;
        n += 1u;
    }
    sink.put8(lo, hi, n);
}

/* ttl: small values dominate (30, 60, 3600 ...), so the four-compare short cut comes first; the branch is
   almost always uniform across a warp */
RG_HD uint32_t ndigits_i32(int32_t v)
{
    const uint32_t u = v < 0 ? 0u - (uint32_t)v : (uint32_t)v;
    const uint32_t neg = v < 0 ? 1u : 0u;
    if (u < 10000u)
        return ndigits4(u) + neg;
    return ndigits_u32(u) + neg;
}

template <class Sink>
RG_HD void put_i32_dec(int32_t v, Sink &sink)
{
    uint32_t u = (uint32_t)v;
    if (v < 0) {
        sink.put1('-');
        u = 0u - u;
    }
    put_u32_dec(u, sink);
}

/* Address fence on a word of address bytes (masked to its valid bytes): every byte
 * must be in 0x20..0x7f and must not be '"' or '\' (they would need a JSON escape). */
RG_HD uint32_t addr_word_bad(uint32_t v, uint32_t keep)
{
    uint32_t v7 = v & 0x7F7F7F7Fu;
    uint32_t ctl = zero7(v7 & 0x60606060u);                 /* byte < 0x20 */
    uint32_t q = eq7(v7, 0x22) | eq7(v7, 0x5C);
    return ((v & 0x80808080u) | ((ctl | q) & keep)) != 0;
}

/* Address fence of one record: non-empty (a falsy adminIp means auto-detect upstream, register.js:143) and every byte
 * passes addr_word_bad. */
template <class Src>
RG_HD uint32_t check_addr(const Src &src, uint32_t off, uint32_t al)
{
    if (al == 0)
        return BAD_ADDR_BYTE;
    uint32_t wi = off >> 2;
    const uint32_t sh = (off & 3u) * 8u;
    uint32_t lo = src.word(wi);
    uint32_t bad = 0;
    uint32_t rem = al;
    while (rem) {
        uint32_t nbytes = rem < 4 ? rem : 4;
        uint32_t hi = src.word_hi(wi + 1, sh + 8 * nbytes > 32 || rem > 4);
        uint32_t keep = low_bytes(nbytes);
        bad |= addr_word_bad(funnel_r(lo, hi, sh) & keep, keep);
        lo = hi;
        wi++;
        rem -= nbytes;
    }
    return bad ? (uint32_t)BAD_ADDR_BYTE : 0u;
}

/*
 * The value fence of one record (REGK_BAD_DOMAIN_BYTE | _HOST_BYTE | _ADDR_BYTE | _TYPE_ID), for a batch's flags
 * exactly as the compose kernels apply it: domains only when paths are composed, hostnames only for host nodes,
 * address and type id only when payloads are composed.  Offsets are not checked here (REGK_BAD_TOO_LARGE is the
 * compose kernels' business).  The skip-mode fence pass (regk_skip.cuh) runs this per record.
 */
template <class DSrc, class HSrc, class ASrc>
RG_HD uint32_t fence_record(const DSrc &dom, uint32_t d0, uint32_t L, const HSrc &host, uint32_t h0, uint32_t H,
    const ASrc &addr, uint32_t a0, uint32_t al, uint32_t type_id, uint32_t ntypes, bool alias, bool do_path, bool do_json)
{
    uint32_t bad = 0;
    if (do_path) {
        bad |= scan_domain(dom, d0, L).bad;
        if (!alias)
            bad |= check_host(host, h0, H);
    }
    if (do_json) {
        bad |= check_addr(addr, a0, al);
        if (type_id >= ntypes)
            bad |= BAD_TYPE_ID;
    }
    return bad;
}

/*
 * Per-type fragment table (built on the host by regk_set_types, JSON escaping
 * already applied).  For type T:
 *   f1 = {"type":"T","address":"        f2 = ,"T":{"address":"
 * Fragments start on word boundaries inside `blob`.
 */
struct TypeFrag {
    uint16_t f1_off, f1_len, f2_off, f2_len;                /* byte offsets into the blob (word aligned) */
};
/* Each fragment is stored as 4 pre-shifted variants, back to back, variant k = k zero bytes + the fragment,
 * zero padded to frag_stride_words(len) words: appending it at byte phase k of the output is then a plain
 * word copy (first word OR-ed with the pending bytes) instead of a shift per word. */
RG_HD uint32_t frag_stride_words(uint32_t len)
{
    return (len + 6u) >> 2;                                 /* ceil((len + 3) / 4) */
}

template <class Src, class Sink>
RG_HD void put_aligned(const Src &blob, uint32_t off, uint32_t len, Sink &sink)
{
    uint32_t wi = off >> 2;
    while (len >= 4) {
        sink.put4(blob.word(wi++));
        len -= 4;
    }
    if (len)
        sink.put(blob.word(wi) & low_bytes(len), len);
}

/* generic sinks: the unshifted variant */
template <class Src, class Sink>
RG_HD void put_frag(const Src &blob, uint32_t off, uint32_t len, Sink &sink)
{
    put_aligned(blob, off, len, sink);
}

/*
 * word sink: copy from the variant that matches the sink's byte phase.
 * OVERSHOOT = true copies a fixed MAXW words with no loop and no bounds (garbage lands in the next <= 16
 * bytes, which the caller guarantees belong to the same record and are written later);
 * OVERSHOOT = false stores exactly the completed words.
 */
template <bool OVERSHOOT, uint32_t MAXW, class Src>
RG_HD void put_frag_w(const Src &blob, uint32_t off, uint32_t len, WordSink &sink)
{
    const uint32_t ph = sink.s >> 3;
    const uint32_t src = (off >> 2) + ph * frag_stride_words(len);
    const uint32_t total = ph + len;
    const uint32_t nfull = total >> 2, rem = total & 3u;
    uint32_t *dst = sink.wp;
    const uint32_t first = blob.word(src) | sink.carry;
    if (OVERSHOOT) {
        uint32_t v[MAXW];
        #pragma unroll
        for (uint32_t i = 1; i < MAXW; i++)
            v[i] = blob.word(src + i);
        dst[0] = first;
        #pragma unroll
        for (uint32_t i = 1; i < MAXW; i++)
            dst[i] = v[i];
        sink.carry = rem ? (nfull ? blob.word(src + nfull) : first) : 0u;
    } else {
        if (nfull == 0) {
            sink.carry = first;
            sink.s = total * 8u;
            return;
        }
        dst[0] = first;
        uint32_t i = 1;
        for (; i + 4 <= nfull; i += 4) {                    /* loads first: 4 independent LDS in flight */
            const uint32_t a = blob.word(src + i), b = blob.word(src + i + 1), c = blob.word(src + i + 2),
                           d = blob.word(src + i + 3);
            dst[i] = a;
            dst[i + 1] = b;
            dst[i + 2] = c;
            dst[i + 3] = d;
        }
        for (; i < nfull; i++)
            dst[i] = blob.word(src + i);
        sink.carry = rem ? blob.word(src + nfull) : 0u;
    }
    sink.wp = dst + nfull;
    sink.s = rem * 8u;
}

/* exact copy of a 16..33-byte fragment without a loop: 9 loads, 4 unconditional + 5 predicated stores */
template <class Src>
RG_HD void put_frag_mid(const Src &blob, uint32_t off, uint32_t len, WordSink &sink)
{
    const uint32_t ph = sink.s >> 3;
    const uint32_t src = (off >> 2) + ph * frag_stride_words(len);
    const uint32_t total = ph + len;                        /* 16..36 */
    const uint32_t nfull = total >> 2, rem = total & 3u;    /* nfull in 4..9 */
    uint32_t *dst = sink.wp;
    uint32_t v[9];
    #pragma unroll
    for (uint32_t i = 0; i < 9; i++)
        v[i] = blob.word(src + i);
    dst[0] = v[0] | sink.carry;
    dst[1] = v[1];
    dst[2] = v[2];
    dst[3] = v[3];
    #pragma unroll
    for (uint32_t i = 4; i < 9; i++)
        if (i < nfull)
            dst[i] = v[i];
    sink.carry = rem ? blob.word(src + nfull) : 0u;
    sink.wp = dst + nfull;
    sink.s = rem * 8u;
}

template <class Src>
RG_HD void put_frag(const Src &blob, uint32_t off, uint32_t len, WordSink &sink)
{
    if (len >= 16u && len <= 33u)
        put_frag_mid(blob, off, len, sink);
    else
        put_frag_w<false, 1>(blob, off, len, sink);
}

/* The opening fragment {"type":"T","address":" : at least 24 more bytes of the record always follow it
 * (address, quote, second fragment, address, "}}), so up to 37 bytes it is copied as 10 unconditional words. */
template <class Src, class Sink>
RG_HD void put_frag_first(const Src &blob, uint32_t off, uint32_t len, Sink &sink)
{
    put_frag(blob, off, len, sink);
}

template <class Src>
RG_HD void put_frag_first(const Src &blob, uint32_t off, uint32_t len, WordSink &sink)
{
    if (len <= 37u)
        put_frag_w<true, 10>(blob, off, len, sink);
    else
        put_frag_w<false, 1>(blob, off, len, sink);
}

/* the first (up to) 16 address bytes, from registers (bytes of aw[] beyond n are zero) */
template <class Sink>
RG_HD void put_addr16(const uint32_t (&aw)[4], uint32_t n, Sink &sink)
{
    #pragma unroll
    for (int w = 0; w < 4; w++) {
        if (n >= 4u * (w + 1))
            sink.put4(aw[w]);
        else if (n > 4u * w)
            sink.put(aw[w], n - 4u * w);
    }
}

/* word sink: shift the whole 16-byte register block once, then store what is complete */
RG_HD void put_addr16(const uint32_t (&aw)[4], uint32_t n, WordSink &sink)
{
    const uint32_t sh = sink.s, back = 32u - sh;
    const uint32_t o0 = sink.carry | (aw[0] << sh);
    const uint32_t o1 = funnel_rc(aw[0], aw[1], back);
    const uint32_t o2 = funnel_rc(aw[1], aw[2], back);
    const uint32_t o3 = funnel_rc(aw[2], aw[3], back);
    const uint32_t o4 = funnel_rc(aw[3], 0u, back);
    const uint32_t total = (sh >> 3) + n;
    const uint32_t nfull = total >> 2;                      /* 0..4 */
    uint32_t *dst = sink.wp;
    if (nfull > 0) dst[0] = o0;
    if (nfull > 1) dst[1] = o1;
    if (nfull > 2) dst[2] = o2;
    if (nfull > 3) dst[3] = o3;
    sink.carry = nfull == 0 ? o0 : nfull == 1 ? o1 : nfull == 2 ? o2 : nfull == 3 ? o3 : o4;
    sink.wp = dst + nfull;
    sink.s = (total & 3u) * 8u;
}

RG_HD uint32_t json_length(uint32_t f1_len, uint32_t f2_len, uint32_t al, bool has_ttl, int32_t ttl,
    bool has_ports, uint32_t k, uint32_t port_digits)
{
    /* f1 + A + ('"' | '","ttl":' + ttl) + f2 + A + ('"}}' | '","ports":[' ... ']}}') */
    uint32_t n = f1_len + f2_len + 2 * al + 4;
    if (has_ttl)
        n += 7 + ndigits_i32(ttl);
    if (has_ports)
        n += 11 + port_digits + (k ? k - 1 : 0);
    return n;
}

#define RG_LE4(a, b, c, d) ((uint32_t)(uint8_t)(a) | ((uint32_t)(uint8_t)(b) << 8) | \
    ((uint32_t)(uint8_t)(c) << 16) | ((uint32_t)(uint8_t)(d) << 24))

/*
 * Emit the JSON payload of one host record (A3 + A4):
 *   {"type":"T","address":"A"[,"ttl":N],"T":{"address":"A"[,"ports":[p,...]]}}
 * The address is passed as up to 16 bytes in registers (aw[0..3]); a longer
 * address continues from asrc at byte offset aoff + 16.  ports are read
 * through port(i).
 */
template <class FSrc, class ASrc, class PortFn, class Sink>
RG_HD void emit_json(const FSrc &blob, const TypeFrag &tf, const uint32_t (&aw)[4], const ASrc &asrc,
    uint32_t aoff, uint32_t al, bool has_ttl, int32_t ttl, bool has_ports, uint32_t k, PortFn port,
    Sink &sink)
{
    const uint32_t a16 = al < 16u ? al : 16u;
    put_frag_first(blob, tf.f1_off, tf.f1_len, sink);       /* {"type":"T","address":" */
    put_addr16(aw, a16, sink);
    if (al > 16u)
        copy_bytes<false>(asrc, aoff + 16u, al - 16u, sink);
    if (has_ttl) {
        sink.put4(RG_LE4('"', ',', '"', 't'));              /* ","ttl": */
        sink.put4(RG_LE4('t', 'l', '"', ':'));
        put_i32_dec(ttl, sink);
    } else {
        sink.put1('"');
    }
    put_frag(blob, tf.f2_off, tf.f2_len, sink);             /* ,"T":{"address":" */
    put_addr16(aw, a16, sink);
    if (al > 16u)
        copy_bytes<false>(asrc, aoff + 16u, al - 16u, sink);
    if (has_ports) {
        sink.put4(RG_LE4('"', ',', '"', 'p'));              /* ","ports":[ */
        sink.put4(RG_LE4('o', 'r', 't', 's'));
        sink.put(RG_LE4('"', ':', '[', 0), 3);
        for (uint32_t i = 0; i < k; i++)
            put_port(port(i), i != 0, sink);
        sink.put(RG_LE4(']', '}', '}', 0), 3);
    } else {
        sink.put(RG_LE4('"', '}', '}', 0), 3);
    }
}

/* ---------------------------------------- service records (regk_service.cuh) -- */

/*
 * {"type":"service","service":{"type":"service","service":{<srvce, proto, port, ttl in the caller's key order>}}}
 * - what lib/register.js:58-62 puts at the domain's node (registration.service as asserted at :186-199).
 */
/* append a string literal, four bytes per sink operation (indices are compile-time constants) */
template <class Sink, size_t N>
RG_HD void put_lit(Sink &sink, const char (&lit)[N])
{
    constexpr uint32_t n = (uint32_t)N - 1u;
    #pragma unroll
    for (uint32_t i = 0; i + 4u <= n; i += 4u)
        sink.put4(RG_LE4(lit[i], lit[i + 1], lit[i + 2], lit[i + 3]));
    constexpr uint32_t r = n & 3u, b = n - r;
    if (r == 1u)
        sink.put1((uint8_t)lit[b]);
    else if (r == 2u)
        sink.put(RG_LE4(lit[b], lit[b + 1 < n ? b + 1 : b], 0, 0), 2);
    else if (r == 3u)
        sink.put(RG_LE4(lit[b], lit[b + 1 < n ? b + 1 : b], lit[b + 2 < n ? b + 2 : b], 0), 3);
}

/* length-only twin of the sinks for literals and strings */
struct LenSink {
    uint32_t n;
    RG_HD void put(uint32_t, uint32_t k) { n += k; }
    RG_HD void put4(uint32_t) { n += 4; }
    RG_HD void put8(uint32_t, uint32_t, uint32_t k) { n += k; }
    RG_HD void put1(uint32_t) { n += 1; }
};

/* key ids of key_order: two bits each, first member in bits 0-1 */
enum : uint32_t { KEY_SRVCE = 0, KEY_PROTO = 1, KEY_PORT = 2, KEY_TTL = 3, KEY_ORDER_DEFAULT = 0xE4 /* 3,2,1,0 from the top */ };

RG_HD bool key_order_ok(uint32_t o)
{
    const uint32_t seen = (1u << (o & 3u)) | (1u << ((o >> 2) & 3u)) | (1u << ((o >> 4) & 3u)) | (1u << ((o >> 6) & 3u));
    return seen == 0xFu;
}

/* the strings are copied without their bytes being looked at: `len_only` sinks skip the loads altogether */
template <class Src, class Sink>
RG_HD void emit_service(const Src &ssrc, uint32_t s0, uint32_t sl, const Src &psrc, uint32_t p0, uint32_t pl,
    uint32_t port, int32_t ttl, uint32_t order, Sink &sink, bool len_only)
{
    put_lit(sink, "{\"type\":\"service\",\"service\":{\"type\":\"service\",\"service\":{");
    #pragma unroll 1
    for (uint32_t i = 0; i < 4u; i++) {
        const uint32_t key = (order >> (2u * i)) & 3u;
        if (i)
            sink.put1(',');
        if (key == KEY_SRVCE || key == KEY_PROTO) {
            if (key == KEY_SRVCE)
                put_lit(sink, "\"srvce\":\"");
            else
                put_lit(sink, "\"proto\":\"");
            const uint32_t o = key == KEY_SRVCE ? s0 : p0, l = key == KEY_SRVCE ? sl : pl;
            if (len_only)
                sink.put(0u, l);
            else
                copy_bytes<false>(key == KEY_SRVCE ? ssrc : psrc, o, l, sink);
            sink.put1('"');
        } else if (key == KEY_PORT) {
            put_lit(sink, "\"port\":");
            put_u32_dec(port, sink);
        } else {
            put_lit(sink, "\"ttl\":");
            put_i32_dec(ttl, sink);
        }
    }
    put_lit(sink, "}}}");
}

/* ------------------------------------ setupDirectories (regk_parents.cuh) -- */

/* node (>= 6) posix path.dirname of an absolute path of n >= 1 bytes, as the length of the directory prefix:
   trailing slashes are skipped, the directory ends before the last '/' that precedes the final segment;
   '/' when there is none, '//' when that separator sits at index 1 (reference lib/register.js:118). */
RG_HD uint32_t dirname_len_scan(const uint8_t *p, uint32_t n)
{
    bool matched_slash = true;
    for (uint32_t i = n - 1; i >= 1; --i) {
        if (p[i] == '/') {
            if (!matched_slash)
                return i == 1 ? 2u : i;
        } else {
            matched_slash = false;
        }
    }
    return 1;
}

/* The same for a host node whose last segment is a hostname of H bytes (non-empty, no '/': the fence): the
   separator in front of it is the one dirname stops at, so no scan is needed. */
RG_HD uint32_t dirname_len_host(uint32_t n, uint32_t H)
{
    const uint32_t d = n - H - 1u;
    return d ? d : 1u;
}

/* k-th 4-byte group of the byte string that starts at byte `o` of the word array W (readable one word past it) */
RG_HD uint32_t string_word(const uint32_t *W, uint64_t o, uint32_t k)
{
    const uint64_t b = (o >> 2) + k;
    return funnel_r(W[b], W[b + 1], ((uint32_t)o & 3u) * 8u);
}

/* one 4-byte group into a running string hash, and the finaliser (murmur3) */
RG_HD uint32_t hash32_step(uint32_t h, uint32_t w)
{
    w *= 0xCC9E2D51u;
    w = (w << 15) | (w >> 17);
    w *= 0x1B873593u;
    h ^= w;
    h = (h << 13) | (h >> 19);
    return h * 5u + 0xE6546B64u;
}

RG_HD uint32_t hash32_final(uint32_t h)
{
    h ^= h >> 16;
    h *= 0x85EBCA6Bu;
    h ^= h >> 13;
    h *= 0xC2B2AE35u;
    h ^= h >> 16;
    return h;
}

/* 32-bit hash of the n bytes at byte offset o (murmur3 mixing, word-wise; only picks a table slot) */
RG_HD uint32_t string_hash32(const uint32_t *W, uint64_t o, uint32_t n)
{
    uint32_t h = 0x9747B28Cu ^ n;
    const uint32_t nw = n >> 2, rem = n & 3u;
    for (uint32_t k = 0; k < nw + (rem ? 1u : 0u); k++) {
        uint32_t w = string_word(W, o, k);
        if (k == nw)
            w &= low_bytes(rem);
        h = hash32_step(h, w);
    }
    return hash32_final(h);
}

/* do the n bytes at byte offsets a and b of W agree? */
RG_HD bool string_equal(const uint32_t *W, uint64_t a, uint64_t b, uint32_t n)
{
    const uint32_t nw = n >> 2, rem = n & 3u;
    for (uint32_t k = 0; k < nw; k++)
        if (string_word(W, a, k) != string_word(W, b, k))
            return false;
    if (rem)
        return ((string_word(W, a, nw) ^ string_word(W, b, nw)) & low_bytes(rem)) == 0u;
    return true;
}

/* ---- the same on a buffer with no slack behind it (a caller's device stream ends where it ends) ---- */

/* word b of W, where only bytes [0, limit) of the buffer may be read: bytes at or past `limit` read as 0 */
RG_HD uint32_t word_clamped(const uint32_t *W, uint64_t b, uint64_t limit)
{
    const uint64_t byte0 = b << 2;
    if (byte0 + 4u <= limit)
        return W[b];
    const uint8_t *B = reinterpret_cast<const uint8_t *>(W);
    uint32_t v = 0;
    for (uint32_t i = 0; i < 4u && byte0 + i < limit; i++)
        v |= (uint32_t)B[byte0 + i] << (8u * i);
    return v;
}

/* string_word with every read below `limit`: equal to string_word for the bytes of a string that ends by `limit` */
RG_HD uint32_t string_word_clamped(const uint32_t *W, uint64_t o, uint32_t k, uint64_t limit)
{
    const uint64_t b = (o >> 2) + k;
    return funnel_r(word_clamped(W, b, limit), word_clamped(W, b + 1u, limit), ((uint32_t)o & 3u) * 8u);
}

/* string_hash32 of the n bytes at o of a buffer readable below `limit`: the same value for the same bytes */
RG_HD uint32_t string_hash32_clamped(const uint32_t *W, uint64_t o, uint32_t n, uint64_t limit)
{
    uint32_t h = 0x9747B28Cu ^ n;
    const uint32_t nw = n >> 2, rem = n & 3u;
    for (uint32_t k = 0; k < nw + (rem ? 1u : 0u); k++) {
        uint32_t w = string_word_clamped(W, o, k, limit);
        if (k == nw)
            w &= low_bytes(rem);
        h = hash32_step(h, w);
    }
    return hash32_final(h);
}

/* do the n bytes at a of buffer A (readable below la) and at b of buffer B (readable below lb) agree? */
RG_HD bool string_equal2(const uint32_t *A, uint64_t a, uint64_t la, const uint32_t *B, uint64_t b, uint64_t lb, uint32_t n)
{
    const uint32_t nw = n >> 2, rem = n & 3u;
    for (uint32_t k = 0; k < nw; k++)
        if (string_word_clamped(A, a, k, la) != string_word_clamped(B, b, k, lb))
            return false;
    if (rem)
        return ((string_word_clamped(A, a, nw, la) ^ string_word_clamped(B, b, nw, lb)) & low_bytes(rem)) == 0u;
    return true;
}

/* ------------------------------------------- the mkdirp set (regk_mkdirp.cuh) -- */

constexpr uint32_t MKDIR_INVALID = 0xFFFFFFFFu;
constexpr uint32_t MKDIR_HASH_SEED = 0x811C9DC5u;

/* What mkdirp(D) creates for a directory D of L bytes, as its number of components: 0 for "/" (or an empty
   directory: nothing to create), MKDIR_INVALID when ZooKeeper's path check would reject D - no leading '/', an
   empty component ("//"), a trailing '/', or a byte in 0x00-0x1F or 0x7F (bytes >= 0x80 and '.' / '..' components
   are outside the domain fence) - else the number of '/' in D. */
RG_HD uint32_t mkdir_components(const uint8_t *p, uint32_t L)
{
    if (L == 0u)
        return 0u;
    if (p[0] != '/')
        return MKDIR_INVALID;
    if (L == 1u)
        return 0u;
    if (p[L - 1u] == '/')
        return MKDIR_INVALID;
    uint32_t depth = 0;
    uint8_t prev = 0;
    for (uint32_t i = 0; i < L; i++) {
        const uint8_t c = p[i];
        if (c < 0x20u || c == 0x7Fu || (c == '/' && prev == '/'))
            return MKDIR_INVALID;
        depth += c == '/' ? 1u : 0u;
        prev = c;
    }
    return depth;
}

/* One more component of a valid directory of L bytes: the prefix that ends at `pos` (0, or a '/' of the directory)
   is extended through the next '/' or the end.  Returns the new prefix length; *h carries the running FNV-1a state
   of the prefix bytes, so that every ancestor's hash costs only its own last component. */
RG_HD uint32_t mkdir_extend(const uint8_t *p, uint32_t pos, uint32_t L, uint32_t *h)
{
    uint32_t s = *h, k = pos;
    do {
        s = (s ^ p[k]) * 0x01000193u;
        k++;
    } while (k < L && p[k] != '/');
    *h = s;
    return k;
}

/* table slot hash of a prefix of L bytes whose running state is h (murmur3 finaliser) */
RG_HD uint32_t mkdir_slot_hash(uint32_t h, uint32_t L)
{
    h ^= L;
    h ^= h >> 16;
    h *= 0x85EBCA6Bu;
    h ^= h >> 13;
    h *= 0xC2B2AE35u;
    h ^= h >> 16;
    return h;
}

}  /* namespace regk */
#endif /* REGK_CORE_CUH */
