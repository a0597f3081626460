/*
 * regk_dns_ptr.cuh — PTR answers for in-addr.arpa names (include/regk.h regk_dns_answer with REGK_DNS_PTR): a reverse
 * index of the resolve's host addresses, and the parse and emit_rr passes of regk_dns.cuh with a third kind of owner.
 *
 * The reverse-name recogniser and the PTR truncation cut are host + device code: tests/emul/dns_ptr_emul.cpp runs them
 * under AddressSanitizer.  The passes (regk_api.cu regk_dns_answer):
 *   index       once per resolve, after regk_dns_prep_kernel wrote ip4: the REGK_Q_HOST_A nodes compacted in node order
 *               (count / compact, the two-level totals of regk_resolve.cuh), their (address, node) pairs sorted by a
 *               stable radix sort (equal addresses stay in node order), the exclusive prefix of PTR RR bytes over the
 *               sorted positions (len / scan)
 *   parse_ptr   regk_dns.cuh's parse body with DnsRev: a reverse name's targets are the sorted positions of its
 *               address (lower / upper bound), cut by whole positions
 *   emit_rr_ptr regk_dns.cuh's emit_rr body with DnsRev: PTR RR t of a response is sorted position first + t
 */
#ifndef REGK_DNS_PTR_CUH
#define REGK_DNS_PTR_CUH

#include "regk_dns.cuh"

namespace regk {

constexpr uint32_t DNS_PTR_RR = 14;             /* pointer owner, type, class, TTL, RDLENGTH, + the name's L + 2 */

/* The address of a reverse name: 6 labels o4.o3.o2.o1.in-addr.arpa of a wire name q that parsed (rules 1-8), each
   octet 1-3 digits without a leading zero and at most 255, the last two labels compared case-insensitively: o1.o2.o3.o4
   big-endian, or DNS_NOT_REVERSE */
constexpr uint64_t DNS_NOT_REVERSE = ~0ull;

RG_HD uint64_t dns_reverse(const uint8_t *q, uint32_t labels)
{
    if (labels != 6u)
        return DNS_NOT_REVERSE;
    uint32_t i = 0, v = 0;
    for (uint32_t k = 0; k < 4; k++) {
        const uint32_t b = q[i];
        if (b < 1u || b > 3u || (b > 1u && q[i + 1] == '0'))
            return DNS_NOT_REVERSE;
        uint32_t o = 0;
        for (uint32_t j = 1; j <= b; j++) {
            const uint32_t c = q[i + j];
            if (c < '0' || c > '9')
                return DNS_NOT_REVERSE;
            o = o * 10u + (c - '0');
        }
        if (o > 255u)
            return DNS_NOT_REVERSE;
        v |= o << (8u * k);
        i += b + 1u;
    }
    if (!dns_label_eq(q + i + 1, q[i], (const uint8_t *)"in-addr", 7u))
        return DNS_NOT_REVERSE;
    i += q[i] + 1u;
    if (!dns_label_eq(q + i + 1, q[i], (const uint8_t *)"arpa", 4u))
        return DNS_NOT_REVERSE;
    return v;
}

/* What of the PTR RRs at sorted positions [f, e) fits in `room` bytes (B: the exclusive prefix of their bytes):
   whole RRs, no additionals */
RG_HD DnsFit dns_fit_ptr(const unsigned long long *B, uint32_t f, uint32_t e, uint32_t room)
{
    DnsFit r;
    const uint32_t c = dns_upper(B, f, e, room);
    r.nans = c - f;
    r.ans_bytes = (uint32_t)(B[c] - B[f]);
    r.nadd = 0;
    r.tc = c < e;
    return r;
}

/* a PTR RR to the dotted name t of tn bytes: owner 0xC00C, the uncompressed name (RFC 1035 3.3.12): 14 + tn bytes */
RG_HD void dns_put_ptr(uint8_t *o, uint32_t ttl, const uint8_t *t, uint32_t tn)
{
    o = dns_put16(o, 0xC00Cu);
    o = dns_put16(o, 12);
    o = dns_put16(o, 1);
    o = dns_put32(o, ttl);
    o = dns_put16(o, tn + 2u);
    dns_put_name(o, t, tn);
}

}  /* namespace regk */

#if defined(__CUDACC__)
namespace regk {

/* the reverse index: n host nodes, their addresses (key) and nodes (val) by address then node, the exclusive prefix
   of their PTR RR bytes [n + 1]; the build's inputs (unsorted pairs), tile totals and count */
struct DnsPtrParams {
    uint64_t n;
    const uint32_t *key, *val;
    const unsigned long long *bytes;
    uint32_t *key_in, *val_in;
    uint32_t *skey, *sval;                      /* key, val writable for the build */
    unsigned long long *sbytes;
    unsigned long long *htile[3], *hsuper[3];   /* [0]: host nodes per tile */
    unsigned long long *btile[3], *bsuper[3];   /* [0]: PTR bytes per tile */
    unsigned long long *count;                  /* [1] host nodes */
};

/* the first sorted position whose address is >= a, or > a when `after` */
__device__ __forceinline__ uint32_t dns_ptr_bound(const uint32_t *key, uint32_t n, uint32_t a, bool after)
{
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        const uint32_t mid = lo + (hi - lo) / 2u;
        if (key[mid] < a || (after && key[mid] == a))
            lo = mid + 1u;
        else
            hi = mid;
    }
    return lo;
}

/* the reverse index as regk_dns.cuh's parse and emit_rr bodies ask for it */
struct DnsRev {
    static constexpr bool on = true;
    static constexpr uint32_t kind_mask = 7u;
    const uint32_t *key, *val;
    const unsigned long long *bytes;
    uint32_t n;

    __device__ DnsSpan owner(const uint8_t *msg, const DnsMsg &r) const
    {
        const uint64_t a = dns_reverse(msg + 12, r.labels);
        if (a == DNS_NOT_REVERSE)
            return DnsSpan{0, 0};
        const uint32_t f = dns_ptr_bound(key, n, (uint32_t)a, false);
        return DnsSpan{f, f < n && key[f] == (uint32_t)a ? dns_ptr_bound(key, n, (uint32_t)a, true) : f};
    }
    __device__ uint64_t node(uint32_t f) const { return val[f]; }
    __device__ DnsFit fit(uint32_t f, uint32_t e, uint32_t room) const { return dns_fit_ptr(bytes, f, e, room); }
    /* PTR RR t of the response answered by node s (the smallest target of its address) at o, the answers' start */
    __device__ void emit(const DnsParams &p, uint8_t *o, uint64_t s, uint32_t t) const
    {
        const uint32_t f = dns_ptr_bound(key, n, p.ip4[s], false), j = f + t, c = val[j];
        dns_put_ptr(o + (bytes[j] - bytes[f]), (uint32_t)p.ttl[c], p.dom + p.path_off[c], p.dec[c].dom_len);
    }
};

/* ---- index: host nodes per tile ---- */
__global__ void __launch_bounds__(RV_TILE) regk_dns_ptr_count_kernel(const DnsParams p, const DnsPtrParams x)
{
    const uint64_t i = (uint64_t)blockIdx.x * RV_TILE + threadIdx.x;
    unsigned long long v[1] = {i < p.m && (p.roles[i] & RV_ROLE_HOST_A) ? 1ull : 0ull}, tot[1];
    rv_block_scan<1>(v, tot);
    if (threadIdx.x == 0)
        rv_add_total(x.htile[0], x.hsuper[0], blockIdx.x, tot[0]);
}

/* ---- index: the host nodes' (address, node) pairs in node order, and their count ---- */
__global__ void __launch_bounds__(RV_TILE) regk_dns_ptr_compact_kernel(const DnsParams p, const DnsPtrParams x)
{
    const uint64_t i = (uint64_t)blockIdx.x * RV_TILE + threadIdx.x;
    unsigned long long base[1], tot[1];
    rv_tile_bases<1>(x.htile, x.hsuper, blockIdx.x, base);
    const bool h = i < p.m && (p.roles[i] & RV_ROLE_HOST_A);
    unsigned long long v[1] = {h ? 1ull : 0ull};
    rv_block_scan<1>(v, tot);
    if (h) {
        x.key_in[base[0] + v[0]] = p.ip4[i];
        x.val_in[base[0] + v[0]] = (uint32_t)i;
    }
    if (i + 1 == p.m)
        x.count[0] = base[0] + v[0] + (h ? 1ull : 0ull);
}

/* ---- index: PTR RR bytes per tile of sorted positions ---- */
__global__ void __launch_bounds__(RV_TILE) regk_dns_ptr_len_kernel(const DnsParams p, const DnsPtrParams x)
{
    const uint64_t j = (uint64_t)blockIdx.x * RV_TILE + threadIdx.x;
    unsigned long long v[1] = {j < x.n ? DNS_PTR_RR + (unsigned long long)p.dec[x.val[j]].dom_len : 0ull}, tot[1];
    rv_block_scan<1>(v, tot);
    if (threadIdx.x == 0)
        rv_add_total(x.btile[0], x.bsuper[0], blockIdx.x, tot[0]);
}

/* ---- index: the exclusive prefix of PTR RR bytes [n + 1] ---- */
__global__ void __launch_bounds__(RV_TILE) regk_dns_ptr_scan_kernel(const DnsParams p, const DnsPtrParams x)
{
    const uint64_t j = (uint64_t)blockIdx.x * RV_TILE + threadIdx.x;
    unsigned long long base[1], tot[1];
    rv_tile_bases<1>(x.btile, x.bsuper, blockIdx.x, base);
    const unsigned long long own = j < x.n ? DNS_PTR_RR + (unsigned long long)p.dec[x.val[j]].dom_len : 0ull;
    unsigned long long v[1] = {own};
    rv_block_scan<1>(v, tot);
    if (j < x.n) {
        x.sbytes[j] = base[0] + v[0];
        if (j + 1 == x.n)
            x.sbytes[x.n] = base[0] + v[0] + own;
    }
}

__device__ __forceinline__ DnsRev dns_rev(const DnsPtrParams &x)
{
    return DnsRev{x.key, x.val, x.bytes, (uint32_t)x.n};
}

/* ---- parse with reverse names (RV_TILE threads; a 64-register ceiling in place of __launch_bounds__, under which
   ptxas settles on 40 registers and spills the reverse-name state around the SRV cut's 64-bit division call) ---- */
__global__ void __maxnreg__(64) regk_dns_parse_ptr_kernel(const DnsParams p, const DnsPtrParams x)
{
    dns_parse_body(p, dns_rev(x));
}

/* ---- emit_rr with PTR RRs ---- */
__global__ void __launch_bounds__(256) regk_dns_emit_rr_ptr_kernel(const DnsParams p, unsigned long long n_rr, const DnsPtrParams x)
{
    dns_emit_rr_body(p, n_rr, dns_rev(x));
}

}  /* namespace regk */
#endif /* __CUDACC__ */
#endif /* REGK_DNS_PTR_CUH */
