/*
 * regk_dns.cuh — DNS responses from a resolved snapshot (include/regk.h regk_dns_answer): a batch of RFC 1035 query
 * messages in, wire-format responses out, answered against the state the last regk_resolve left on the device (its
 * path table, classes, roles, TTLs, decoded records and the children grouped by service).
 *
 * The per-message rules (the parser, the question's path, the SRV label match and the truncation arithmetic) are host
 * + device code: tests/emul/dns_emul.cpp runs them under AddressSanitizer.  The passes (regk_api.cu regk_dns_answer):
 *   prep        once per resolve: per node its IPv4 address; per sorted child position the SRV wire bytes, SRV RRs
 *               and additional RRs, with per-tile totals (two-level totals of regk_resolve.cuh)
 *   prep_scan   exclusive prefixes of the three over the sorted positions
 *   check       device input: the smallest message whose offsets are bad, before any message byte is read
 *   parse       one thread per message: the rules, the lower-cased path of the question name into a scratch copy at
 *               the message's own offset, the table probes (the SRV service path is a prefix of the same path), the
 *               truncation cut; per-tile totals of response bytes and RRs, status counts
 *   place       resp_off and the first RR of every response
 *   emit_head   one thread per response: header, echoed question, OPT
 *   emit_rr     one thread per RR, at its closed-form offset: its response by a binary search over the RR bases, its
 *               child and port by binary searches over the service's prefixes
 */
#ifndef REGK_DNS_CUH
#define REGK_DNS_CUH

#include "regk_resolve.cuh"

namespace regk {

enum : uint8_t { DNS_ANSWER = 0, DNS_NODATA = 1, DNS_NXDOMAIN = 2, DNS_FORMERR = 3, DNS_NOTIMP = 4, DNS_REFUSED = 5,
                 DNS_BADVERS = 6, DNS_DROPPED = 7 };               /* include/regk.h REGK_DNS_* */
enum : uint32_t { DNS_K_NONE = 0, DNS_K_HOST_A = 1, DNS_K_SERVICE_A = 2, DNS_K_SRV = 3,
                  DNS_K_PTR = 4 };                  /* regk_dns_ptr.cuh: meta's kind field is 3 bits there */
constexpr uint32_t DNS_A_RR = 16;               /* pointer owner, type, class, TTL, RDLENGTH, IPv4 */
constexpr uint32_t DNS_OPT_RR = 11;
constexpr uint32_t DNS_PTR_MAX = 0x3FFF;        /* a compression pointer's reach (RFC 1035 4.1.4) */

RG_HD uint32_t dns_u16(const uint8_t *m, uint32_t i)
{
    return (uint32_t)m[i] << 8 | m[i + 1];
}

RG_HD bool dns_plain(uint8_t c)
{
    return (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z') || (c >= '0' && c <= '9') || c == '_' || c == '-';
}

RG_HD uint8_t dns_lower(uint8_t c)
{
    return c >= 'A' && c <= 'Z' ? (uint8_t)(c + 32) : c;
}

/* What rules 1-8 (include/regk.h) make of one message of n bytes */
struct DnsMsg {
    uint32_t status;                            /* DNS_*; DNS_ANSWER: the lookup decides */
    uint32_t qend;                              /* end of the question (12 + name + 4) when it parsed */
    uint32_t name, labels;                      /* wire bytes of the question name (root byte included), its labels */
    uint32_t qtype, qclass;
    uint32_t opt, dobit, req_size;              /* an OPT record, its DO bit and its CLASS */
    uint32_t plain;                             /* every label byte in [A-Za-z0-9_-] */
};

RG_HD DnsMsg dns_parse(const uint8_t *m, uint32_t n)
{
    DnsMsg r;
    r.status = DNS_FORMERR;
    r.qend = r.name = r.labels = r.qtype = r.qclass = r.opt = r.dobit = r.req_size = 0;
    r.plain = 1;
    if (n < 12u || (m[2] & 0x80u)) {
        r.status = DNS_DROPPED;
        return r;
    }
    if ((m[2] >> 3) & 15u) {
        r.status = DNS_NOTIMP;
        return r;
    }
    const uint32_t ar = dns_u16(m, 10);
    if (dns_u16(m, 4) != 1u || dns_u16(m, 6) || dns_u16(m, 8) || ar > 1u)
        return r;
    uint32_t i = 12;
    for (;;) {
        if (i >= n || i - 12u >= 255u)
            return r;                           /* past the message, or a 256th name byte */
        const uint32_t b = m[i++];
        if (b & 0xC0u)
            return r;                           /* a compression pointer or an extended label type */
        if (b == 0)
            break;
        if (i + b > n)
            return r;
        for (uint32_t k = 0; k < b; k++)
            r.plain &= dns_plain(m[i + k]) ? 1u : 0u;
        i += b;
        r.labels++;
    }
    r.name = i - 12u;
    if (i + 4u > n)
        return r;
    r.qtype = dns_u16(m, i);
    r.qclass = dns_u16(m, i + 2);
    i += 4;
    r.qend = i;
    uint32_t version = 0;
    if (ar) {                                   /* OPT: root owner, TYPE 41, RDATA inside the message */
        if (i + 11u > n || m[i] != 0 || dns_u16(m, i + 1) != 41u)
            return r;
        r.opt = 1;
        r.req_size = dns_u16(m, i + 3);
        version = m[i + 6];
        r.dobit = m[i + 7] >> 7;
        const uint32_t rdlen = dns_u16(m, i + 9);
        i += 11;
        if (i + rdlen > n)
            return r;
        i += rdlen;
    }
    if (i != n)
        return r;                               /* bytes after the last record */
    r.status = version ? DNS_BADVERS : r.qclass != 1u ? DNS_REFUSED : DNS_ANSWER;
    return r;
}

/* The lower-cased path of a wire name of `labels` labels at q ('/' + the labels in reverse order, joined by '/') into
   out; returns its length (the name's wire bytes - 1).  The path without the first two labels is its prefix. */
RG_HD uint32_t dns_path(const uint8_t *q, uint32_t name, uint8_t *out)
{
    uint32_t e = name - 1u, i = 0;
    for (uint32_t b = q[0]; b; b = q[i]) {
        out[e - b - 1u] = '/';
        for (uint32_t k = 0; k < b; k++)
            out[e - b + k] = dns_lower(q[i + 1u + k]);
        e -= b + 1u;
        i += b + 1u;
    }
    return name - 1u;
}

/* label bytes [l, l + n) equal s[0, sn) ASCII case-insensitively */
RG_HD bool dns_label_eq(const uint8_t *l, uint32_t n, const uint8_t *s, uint32_t sn)
{
    if (n != sn)
        return false;
    for (uint32_t k = 0; k < n; k++)
        if (dns_lower(l[k]) != dns_lower(s[k]))
            return false;
    return true;
}

RG_HD uint32_t dns_limit(bool tcp, uint32_t opt, uint32_t req_size, uint32_t udp_payload)
{
    if (tcp)
        return 65535u;
    if (!opt)
        return 512u;
    return req_size < 512u ? 512u : req_size > udp_payload ? udp_payload : req_size;
}

/* largest c in [f, e] with X[c] - X[f] <= v (X nondecreasing) */
RG_HD uint32_t dns_upper(const unsigned long long *X, uint32_t f, uint32_t e, unsigned long long v)
{
    uint32_t lo = f, hi = e;
    while (lo < hi) {
        const uint32_t mid = lo + (hi - lo + 1u) / 2u;
        if (X[mid] - X[f] <= v)
            lo = mid;
        else
            hi = mid - 1u;
    }
    return lo;
}

struct DnsFit {
    uint32_t nans, nadd, ans_bytes, tc;
};

struct DnsSpan {
    uint32_t f, e;                              /* positions [f, e) */
};

/* What of a query's RRs fits in L bytes after `base` bytes of header, question and OPT.  A host A: one RR.  A service
   (children at sorted positions [f, e)): A, one RR per child; SRV, the prefixes S (SRV bytes), N (SRV RRs) and A
   (additional RRs) over the sorted positions, whose cut-off child and port come from a binary search and a division.
   Additionals only when every answer fit, and only those whose owner pointer (the target name at SRV RR + 18, the
   answers starting at qend) is within a pointer's reach. */
RG_HD DnsFit dns_fit(uint32_t kind, uint32_t f, uint32_t e, const unsigned long long *S, const unsigned long long *N,
    const unsigned long long *A, uint32_t L, uint32_t base, uint32_t qend)
{
    DnsFit r;
    r.nans = r.nadd = r.ans_bytes = r.tc = 0;
    const uint32_t room = L - base;
    if (kind == DNS_K_HOST_A || kind == DNS_K_SERVICE_A) {
        const uint32_t all = kind == DNS_K_HOST_A ? 1u : e - f, fit = room / DNS_A_RR;
        r.nans = all < fit ? all : fit;
        r.ans_bytes = r.nans * DNS_A_RR;
        r.tc = r.nans < all;
        return r;
    }
    if (kind != DNS_K_SRV)
        return r;
    const uint32_t c = dns_upper(S, f, e, room);
    uint32_t bytes = (uint32_t)(S[c] - S[f]), rrs = (uint32_t)(N[c] - N[f]);
    if (c < e) {                                /* child c is cut: whole ports of it */
        const uint32_t unit = (uint32_t)((S[c + 1] - S[c]) / (N[c + 1] - N[c]));
        const uint32_t k = (room - bytes) / unit;
        bytes += k * unit;
        rrs += k;
        r.tc = 1;
    }
    r.nans = rrs;
    r.ans_bytes = bytes;
    if (r.tc)
        return r;
    const uint32_t reach = dns_upper(S, f, e, DNS_PTR_MAX - 18u - qend);
    const uint32_t cend = reach < e ? reach + 1u : e;
    const uint32_t all = (uint32_t)(A[cend] - A[f]), fit = (room - bytes) / DNS_A_RR;
    r.nadd = all < fit ? all : fit;
    return r;
}

/* response bytes of a message: nothing when dropped, the header alone for FORMERR / NOTIMP */
RG_HD uint32_t dns_resp_len(uint32_t status, uint32_t qend, uint32_t opt, uint32_t ans_bytes, uint32_t nadd)
{
    if (status == DNS_DROPPED)
        return 0;
    if (status == DNS_FORMERR || status == DNS_NOTIMP)
        return 12u;
    return qend + ans_bytes + nadd * DNS_A_RR + (opt ? DNS_OPT_RR : 0u);
}

/* dotted-quad text (rv_ipv4_ok) as a big-endian address */
RG_HD uint32_t dns_ipv4(const uint8_t *p, uint32_t n)
{
    uint32_t a = 0, v = 0;
    for (uint32_t k = 0; k < n; k++) {
        if (p[k] == '.') {
            a = a << 8 | v;
            v = 0;
        } else {
            v = v * 10u + (uint32_t)(p[k] - '0');
        }
    }
    return a << 8 | v;
}

RG_HD uint8_t *dns_put16(uint8_t *o, uint32_t v)
{
    o[0] = (uint8_t)(v >> 8);
    o[1] = (uint8_t)v;
    return o + 2;
}

RG_HD uint8_t *dns_put32(uint8_t *o, uint32_t v)
{
    o = dns_put16(o, v >> 16);
    return dns_put16(o, v & 0xFFFFu);
}

/* an A RR: owner pointer, TTL, address */
RG_HD void dns_put_a(uint8_t *o, uint32_t owner, uint32_t ttl, uint32_t addr)
{
    o = dns_put16(o, 0xC000u | owner);
    o = dns_put16(o, 1);
    o = dns_put16(o, 1);
    o = dns_put32(o, ttl);
    o = dns_put16(o, 4);
    dns_put32(o, addr);
}

/* the dotted name t of tn bytes as an uncompressed wire name of tn + 2 bytes */
RG_HD void dns_put_name(uint8_t *o, const uint8_t *t, uint32_t tn)
{
    uint8_t *len = o++;
    uint32_t run = 0;
    for (uint32_t k = 0; k < tn; k++) {
        if (t[k] == '.') {
            *len = (uint8_t)run;
            len = o++;
            run = 0;
        } else {
            *o++ = t[k];
            run++;
        }
    }
    *len = (uint8_t)run;
    *o = 0;
}

/* an SRV RR to the dotted name t of tn bytes: owner 0xC00C, priority 0, weight 10, port, the uncompressed target */
RG_HD void dns_put_srv(uint8_t *o, uint32_t ttl, uint32_t port, const uint8_t *t, uint32_t tn)
{
    o = dns_put16(o, 0xC00Cu);
    o = dns_put16(o, 33);
    o = dns_put16(o, 1);
    o = dns_put32(o, ttl);
    o = dns_put16(o, 8u + tn);
    o = dns_put16(o, 0);
    o = dns_put16(o, 10);
    o = dns_put16(o, port);
    dns_put_name(o, t, tn);
}

}  /* namespace regk */

#if defined(__CUDACC__)
namespace regk {

/* counters[]: [0] the smallest message with bad offsets (~0 = none), the totals, the status counts */
enum { DNS_C_BAD = 0, DNS_C_RESP = 1, DNS_C_RR = 2, DNS_C_TC = 3, DNS_C_STATUS = 4, DNS_NCOUNTERS = 12 };

struct DnsParams {
    /* the resolve's state */
    uint64_t m;
    const uint8_t *path;
    const unsigned long long *path_off;
    uint64_t path_total;
    const uint8_t *json;
    const unsigned long long *json_off;
    const Decoded *dec;
    const uint8_t *dom;
    const uint32_t *ports;
    uint32_t mask;
    const uint32_t *table;
    const uint8_t *cls, *roles;
    const int32_t *ttl;
    const uint32_t *skey, *sval, *first, *end;
    /* prep: per node its address, per sorted position SRV bytes / SRV RRs / additional RRs, then their prefixes */
    uint32_t *ip4;
    unsigned long long *cum[3];
    unsigned long long *ctile[3], *csuper[3];
    /* the queries */
    uint64_t k;
    const uint8_t *msgs;
    const unsigned long long *off;
    uint64_t total;
    uint8_t *scratch;                           /* [total + 16] the question paths */
    uint32_t udp_payload, tcp;
    uint8_t *status, *tc;                       /* [k] */
    unsigned long long *node;                   /* [k] */
    uint32_t *meta, *nans, *nadd, *ans_bytes;   /* [k] meta: qend | opt << 9 | DO << 10 | kind << 11 */
    unsigned long long *qtile[3], *qsuper[3];   /* two-level totals of response bytes and RRs */
    unsigned long long *resp_off, *rr_base;     /* [k + 1] */
    unsigned long long *counters;
    uint8_t *resp;
};

/* ---- prep: addresses and the per-child wire sizes ---- */
__global__ void __launch_bounds__(RV_TILE) regk_dns_prep_kernel(const DnsParams p)
{
    const uint64_t i = (uint64_t)blockIdx.x * RV_TILE + threadIdx.x;
    unsigned long long b[3] = {0ull, 0ull, 0ull}, tot[3];
    if (i < p.m) {
        if (p.roles[i] & (RV_ROLE_HOST_A | RV_ROLE_CHILD)) {
            const Decoded &d = p.dec[i];
            p.ip4[i] = dns_ipv4(p.json + p.json_off[i] + d.addr_pos, d.addr_len);
        }
        const uint32_t s = p.skey[i];
        if (s < p.m) {
            const uint32_t c = p.sval[i];
            const uint32_t np = p.dec[c].nports != 0xFFFFFFFFu ? p.dec[c].nports : 1u;
            b[0] = (unsigned long long)np * (20u + p.dec[c].dom_len);
            b[1] = np;
            b[2] = np ? 1ull : 0ull;
        }
        #pragma unroll
        for (int k = 0; k < 3; k++)
            p.cum[k][i] = b[k];
    }
    rv_block_scan<3>(b, tot);
    if (threadIdx.x == 0) {
        #pragma unroll
        for (int k = 0; k < 3; k++)
            rv_add_total(p.ctile[k], p.csuper[k], blockIdx.x, tot[k]);
    }
}

__global__ void __launch_bounds__(RV_TILE) regk_dns_prep_scan_kernel(const DnsParams p)
{
    const uint64_t i = (uint64_t)blockIdx.x * RV_TILE + threadIdx.x;
    unsigned long long base[3], v[3], own[3], tot[3];
    rv_tile_bases<3>(p.ctile, p.csuper, blockIdx.x, base);
    #pragma unroll
    for (int k = 0; k < 3; k++)
        own[k] = v[k] = i < p.m ? p.cum[k][i] : 0ull;
    rv_block_scan<3>(v, tot);
    if (i < p.m) {
        #pragma unroll
        for (int k = 0; k < 3; k++) {
            p.cum[k][i] = base[k] + v[k];
            if (i + 1 == p.m)
                p.cum[k][p.m] = base[k] + v[k] + own[k];
        }
    }
}

/* ---- check: device offsets, before any message byte is read ---- */
__global__ void __launch_bounds__(256) regk_dns_check_kernel(const DnsParams p)
{
    const uint64_t i = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= p.k)
        return;
    const unsigned long long o0 = p.off[i], o1 = p.off[i + 1];
    if (o0 > o1 || o1 > p.total || o1 - o0 > 65535ull || (i + 1 == p.k && o1 != p.total))
        atomicMin(p.counters + DNS_C_BAD, (unsigned long long)i);
}

/* the snapshot node whose path is scratch[o, o + n), or ~0 */
__device__ __forceinline__ uint64_t dns_find(const DnsParams &p, unsigned long long o, uint32_t n)
{
    const uint32_t *W = reinterpret_cast<const uint32_t *>(p.scratch), *P = reinterpret_cast<const uint32_t *>(p.path);
    const uint64_t lim = p.total + 16u;
    uint32_t slot = string_hash32_clamped(W, o, n, lim) & p.mask;
    for (;;) {
        const uint32_t cur = p.table[slot];
        if (cur == 0u)
            return ~0ull;
        const uint64_t j = cur - 1u;
        const unsigned long long j0 = p.path_off[j];
        if ((uint32_t)(p.path_off[j + 1] - j0) == n && string_equal2(W, o, lim, P, j0, p.path_total, n))
            return j;
        slot = (slot + 1u) & p.mask;
    }
}

/* No reverse names (regk_dns_parse_kernel, regk_dns_emit_rr_kernel): what the bodies below ask of a reverse index
   (regk_dns_ptr.cuh DnsRev) when `on`, folded away here */
struct DnsNoRev {
    static constexpr bool on = false;
    static constexpr uint32_t kind_mask = 3u;   /* the kind bits of meta these kernels read */
    __device__ DnsSpan owner(const uint8_t *, const DnsMsg &) const { return DnsSpan{0, 0}; }
    __device__ uint64_t node(uint32_t) const { return ~0ull; }
    __device__ DnsFit fit(uint32_t, uint32_t, uint32_t) const { return DnsFit{0, 0, 0, 0}; }
    __device__ void emit(const DnsParams &, uint8_t *, uint64_t, uint32_t) const {}
};

/* ---- parse: rules, lookup and the truncation cut, one thread per message ---- */
template <class Rev>
__device__ __forceinline__ void dns_parse_body(const DnsParams &p, const Rev &rev)
{
    __shared__ unsigned int s_cnt[9];
    const uint64_t i = (uint64_t)blockIdx.x * RV_TILE + threadIdx.x;
    if (threadIdx.x < 9)
        s_cnt[threadIdx.x] = 0;
    __syncthreads();
    unsigned long long v[2] = {0ull, 0ull}, tot[2];
    if (i < p.k) {
        const unsigned long long o0 = p.off[i];
        const uint8_t *msg = p.msgs + o0;
        const DnsMsg r = dns_parse(msg, (uint32_t)(p.off[i + 1] - o0));
        uint32_t status = r.status, kind = DNS_K_NONE;
        unsigned long long node = ~0ull;
        DnsFit fit{0, 0, 0, 0};
        if (status == DNS_ANSWER) {
            uint64_t own_a = ~0ull, own_s = ~0ull;
            if (r.plain && r.labels) {
                const uint32_t n = dns_path(msg + 12, r.name, p.scratch + o0);
                const uint64_t j = dns_find(p, o0, n);
                if (j != ~0ull && (p.roles[j] & (RV_ROLE_HOST_A | RV_ROLE_SERVICE)))
                    own_a = j;
                if (r.labels >= 3u) {
                    const uint32_t l0 = msg[12], l1 = msg[13 + l0];
                    const uint64_t s = dns_find(p, o0, n - l0 - l1 - 2u);
                    if (s != ~0ull && (p.roles[s] & RV_ROLE_SERVICE)) {
                        const Decoded &d = p.dec[s];
                        const uint8_t *sj = p.json + p.json_off[s];
                        if (dns_label_eq(msg + 13, l0, sj + d.type_pos, d.type_len) &&
                            dns_label_eq(msg + 14 + l0, l1, sj + d.addr_pos, d.addr_len))
                            own_s = s;
                    }
                }
            }
            if (r.qtype == 1u && own_a != ~0ull) {
                kind = (p.roles[own_a] & RV_ROLE_HOST_A) ? DNS_K_HOST_A : DNS_K_SERVICE_A;
                node = own_a;
            } else if (r.qtype == 33u && own_s != ~0ull) {
                kind = DNS_K_SRV;
                node = own_s;
            } else {
                /* a reverse name's targets (sorted positions), looked up only where they decide the answer */
                const bool owns = own_a != ~0ull || own_s != ~0ull;
                const DnsSpan pt = Rev::on && (r.qtype == 12u || !owns) ? rev.owner(msg, r) : DnsSpan{0, 0};
                if (Rev::on && r.qtype == 12u && pt.f < pt.e) {
                    kind = DNS_K_PTR;
                    node = rev.node(pt.f);
                    const uint32_t L = dns_limit(p.tcp != 0, r.opt, r.req_size, p.udp_payload);
                    fit = rev.fit(pt.f, pt.e, L - r.qend - (r.opt ? DNS_OPT_RR : 0u));
                } else {
                    status = (owns || pt.f < pt.e) ? DNS_NODATA : DNS_NXDOMAIN;
                }
            }
            if (kind != DNS_K_NONE && (!Rev::on || kind != DNS_K_PTR)) {
                const uint32_t f = kind == DNS_K_HOST_A ? 0u : p.first[node], e = kind == DNS_K_HOST_A ? 0u : p.end[node];
                const uint32_t L = dns_limit(p.tcp != 0, r.opt, r.req_size, p.udp_payload);
                fit = dns_fit(kind, f, e, p.cum[0], p.cum[1], p.cum[2], L, r.qend + (r.opt ? DNS_OPT_RR : 0u), r.qend);
            }
        }
        p.status[i] = (uint8_t)status;
        p.tc[i] = (uint8_t)fit.tc;
        p.node[i] = node;
        p.meta[i] = r.qend | r.opt << 9 | r.dobit << 10 | kind << 11;
        p.nans[i] = fit.nans;
        p.nadd[i] = fit.nadd;
        p.ans_bytes[i] = fit.ans_bytes;
        v[0] = dns_resp_len(status, r.qend, r.opt, fit.ans_bytes, fit.nadd);
        v[1] = (unsigned long long)fit.nans + fit.nadd;
        atomicAdd(s_cnt + status, 1u);
        if (fit.tc)
            atomicAdd(s_cnt + 8, 1u);
    }
    rv_block_scan<2>(v, tot);
    if (threadIdx.x == 0) {
        #pragma unroll
        for (int k = 0; k < 2; k++)
            rv_add_total(p.qtile[k], p.qsuper[k], blockIdx.x, tot[k]);
    }
    if (threadIdx.x < 9 && s_cnt[threadIdx.x])
        atomicAdd(p.counters + (threadIdx.x < 8 ? DNS_C_STATUS + threadIdx.x : DNS_C_TC), (unsigned long long)s_cnt[threadIdx.x]);
}

__global__ void __launch_bounds__(RV_TILE) regk_dns_parse_kernel(const DnsParams p)
{
    dns_parse_body(p, DnsNoRev{});
}

/* ---- place: resp_off and rr_base, and the totals ---- */
__global__ void __launch_bounds__(RV_TILE) regk_dns_place_kernel(const DnsParams p)
{
    const uint64_t i = (uint64_t)blockIdx.x * RV_TILE + threadIdx.x;
    unsigned long long base[2], v[2] = {0ull, 0ull}, own[2], tot[2];
    rv_tile_bases<2>(p.qtile, p.qsuper, blockIdx.x, base);
    if (i < p.k) {
        const uint32_t meta = p.meta[i];
        v[0] = dns_resp_len(p.status[i], meta & 511u, (meta >> 9) & 1u, p.ans_bytes[i], p.nadd[i]);
        v[1] = (unsigned long long)p.nans[i] + p.nadd[i];
    }
    own[0] = v[0];
    own[1] = v[1];
    rv_block_scan<2>(v, tot);
    if (i >= p.k)
        return;
    p.resp_off[i] = base[0] + v[0];
    p.rr_base[i] = base[1] + v[1];
    if (i + 1 == p.k) {
        p.resp_off[p.k] = p.counters[DNS_C_RESP] = base[0] + v[0] + own[0];
        p.rr_base[p.k] = p.counters[DNS_C_RR] = base[1] + v[1] + own[1];
    }
}

/* ---- emit_head: header, the echoed question, OPT ---- */
__global__ void __launch_bounds__(256) regk_dns_emit_head_kernel(const DnsParams p)
{
    const uint64_t i = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= p.k)
        return;
    const uint32_t status = p.status[i];
    if (status == DNS_DROPPED)
        return;
    const uint8_t *msg = p.msgs + p.off[i];
    uint8_t *o = p.resp + p.resp_off[i];
    const bool bare = status == DNS_FORMERR || status == DNS_NOTIMP;
    const uint32_t meta = p.meta[i], qend = meta & 511u, opt = bare ? 0u : (meta >> 9) & 1u;
    const uint32_t rcode = status == DNS_NXDOMAIN ? 3u : status == DNS_FORMERR ? 1u : status == DNS_NOTIMP ? 4u :
        status == DNS_REFUSED ? 5u : 0u;
    const uint32_t aa = status <= DNS_NXDOMAIN ? 4u : 0u;
    o[0] = msg[0];
    o[1] = msg[1];
    o[2] = (uint8_t)(0x80u | (msg[2] & 0x78u) | aa | (p.tc[i] ? 2u : 0u) | (msg[2] & 1u));
    o[3] = (uint8_t)rcode;
    dns_put16(o + 4, bare ? 0u : 1u);
    dns_put16(o + 6, p.nans[i]);
    dns_put16(o + 8, 0);
    dns_put16(o + 10, p.nadd[i] + opt);
    if (bare)
        return;
    for (uint32_t k = 12; k < qend; k++)
        o[k] = msg[k];
    if (opt) {
        uint8_t *t = p.resp + p.resp_off[i + 1] - DNS_OPT_RR;
        t[0] = 0;
        dns_put16(t + 1, 41);
        dns_put16(t + 3, p.udp_payload);
        dns_put32(t + 5, (status == DNS_BADVERS ? 1u << 24 : 0u) | ((meta >> 10) & 1u) << 15);
        dns_put16(t + 9, 0);
    }
}

/* ---- emit_rr: one thread per RR ---- */
template <class Rev>
__device__ __forceinline__ void dns_emit_rr_body(const DnsParams &p, unsigned long long n_rr, const Rev &rev)
{
    const unsigned long long r = (unsigned long long)blockIdx.x * 256 + threadIdx.x;
    if (r >= n_rr)
        return;
    uint64_t lo = 0, hi = p.k - 1;                      /* the last response whose first RR is at or before r */
    while (lo < hi) {
        const uint64_t mid = lo + (hi - lo + 1) / 2;
        if (p.rr_base[mid] <= r)
            lo = mid;
        else
            hi = mid - 1;
    }
    const uint64_t q = lo;
    const uint32_t t = (uint32_t)(r - p.rr_base[q]), meta = p.meta[q], qend = meta & 511u, kind = (meta >> 11) & Rev::kind_mask;
    const uint32_t nans = p.nans[q];
    const uint64_t s = p.node[q];
    uint8_t *o = p.resp + p.resp_off[q] + qend;
    if (kind == DNS_K_HOST_A) {
        dns_put_a(o, 12u, (uint32_t)p.ttl[s], p.ip4[s]);
        return;
    }
    if (Rev::on && kind == DNS_K_PTR) {
        rev.emit(p, o, s, t);
        return;
    }
    const uint32_t f = p.first[s], e = p.end[s];
    const int32_t ts = p.ttl[s];
    if (kind == DNS_K_SERVICE_A) {
        const uint32_t c = p.sval[f + t];
        dns_put_a(o + t * DNS_A_RR, 12u, (uint32_t)min(ts, p.ttl[c]), p.ip4[c]);
        return;
    }
    const unsigned long long *S = p.cum[0], *N = p.cum[1], *A = p.cum[2];
    if (t < nans) {                                     /* SRV RR t: child, port */
        const uint32_t ci = dns_upper(N, f, e, t);
        const uint32_t c = p.sval[ci], kp = t - (uint32_t)(N[ci] - N[f]);
        const Decoded &dc = p.dec[c];
        const bool own = dc.nports != 0xFFFFFFFFu;
        const uint32_t port = own ? p.ports[(p.json_off[c] >> 1) + kp] : p.ports[p.json_off[s] >> 1];
        dns_put_srv(o + (S[ci] - S[f]) + (unsigned long long)kp * (20u + dc.dom_len), (uint32_t)ts, port, p.dom + p.path_off[c],
            dc.dom_len);
        return;
    }
    const uint32_t ta = t - nans;                       /* additional ta: the child of the (ta+1)-th first SRV RR */
    const uint32_t ci = dns_upper(A, f, e, ta), c = p.sval[ci];
    dns_put_a(o + p.ans_bytes[q] + ta * DNS_A_RR, qend + (uint32_t)(S[ci] - S[f]) + 18u, (uint32_t)p.ttl[c], p.ip4[c]);
}

__global__ void __launch_bounds__(256) regk_dns_emit_rr_kernel(const DnsParams p, unsigned long long n_rr)
{
    dns_emit_rr_body(p, n_rr, DnsNoRev{});
}

}  /* namespace regk */
#endif /* __CUDACC__ */
#endif /* REGK_DNS_CUH */
