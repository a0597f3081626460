/*
 * regk_resolve.cuh — what DNS answers for a registry snapshot (include/regk.h regk_resolve; README.md:441-755 of the
 * reference, restricted to the canonical record forms this library writes).  Host records are joined to the service
 * record of their parent directory, filtered by the two type tables (README.md:274-282), expanded per port and given
 * TTLs from both sides; the answers come out as dig presentation lines with single tabs.
 *
 * The per-node rules (classify, name check, IPv4 check, line lengths and line writers) are host + device code:
 * tests/emul/resolve_emul.cpp runs them under AddressSanitizer.  The passes (regk_api.cu regk_resolve), after
 * regk_reconcile_insert_kernel (offsets check, paths into the table) and regk_decode_kernel (host_nodes = 0):
 *   classify     one thread per node: duplicate path, class, roles, TTL
 *   join         one thread per candidate child: its parent prefix probes the table read-only; the key is the
 *                service node it belongs to (m: none)
 *   sort         a stable radix sort of (key, node) groups each service's children in node order
 *   child_len    one thread per sorted position: the bytes of the child's A line, SRV lines and additional line, the
 *                service's range [first, end) of sorted positions; per-tile totals
 *   child_scan   exclusive prefixes of the three byte counts over the sorted positions (two-level totals)
 *   qlen / place one thread per node: queries, section bytes, unresolved flag; per-tile totals, then q_kind, q_node,
 *                sec_off and the unresolved list
 *   emit         one thread per HOST_A node, one per child (its A line, SRV lines, additional line), each at its
 *                section's base plus the child's prefix inside the service
 */
#ifndef REGK_RESOLVE_CUH
#define REGK_RESOLVE_CUH

#include "regk_decode_core.cuh"

namespace regk {

enum : uint8_t { RV_OK = 0, RV_EMPTY = 1, RV_NOT_RECORD = 2, RV_BAD_NAME = 3, RV_UNKNOWN_TYPE = 4, RV_BAD_ADDRESS = 5,
                 RV_BAD_TTL = 6, RV_BAD_PORT = 7 };                 /* include/regk.h REGK_RSV_* */
enum : uint8_t { RV_ROLE_HOST_A = 1, RV_ROLE_SERVICE = 2, RV_ROLE_CHILD = 4 };
enum : uint8_t { RV_Q_HOST_A = 1, RV_Q_SERVICE_A = 2, RV_Q_SERVICE_SRV = 3 };  /* REGK_Q_* */

/* bytes [p, p + n) spell s */
RG_HD bool rv_eq(const uint8_t *p, uint32_t n, const char *s)
{
    uint32_t k = 0;
    for (; s[k]; k++)
        if (k >= n || p[k] != (uint8_t)s[k])
            return false;
    return k == n;
}

/* README.md:274-282, compared raw: bit 0 answers a direct query, bit 1 backs a service, 0 unknown */
RG_HD uint32_t rv_type_roles(const uint8_t *t, uint32_t n)
{
    if (rv_eq(t, n, "db_host") || rv_eq(t, n, "host"))
        return 1u;
    if (rv_eq(t, n, "load_balancer") || rv_eq(t, n, "moray_host") || rv_eq(t, n, "redis_host"))
        return 3u;
    if (rv_eq(t, n, "ops_host") || rv_eq(t, n, "rr_host"))
        return 2u;
    return 0u;
}

/* A DNS name fed byte by byte: every label 1-63 bytes of [A-Za-z0-9_-], at most 253 bytes in all */
struct RvName {
    uint32_t label, total;
    bool ok;
    RG_HD void init()
    {
        label = total = 0;
        ok = true;
    }
    RG_HD void feed(uint8_t c)
    {
        if (c == '.') {
            ok = ok && label != 0;
            label = 0;
        } else {
            const bool v = (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z') || (c >= '0' && c <= '9') || c == '_' || c == '-';
            label++;
            ok = ok && v && label <= 63u;
        }
        total++;
    }
    RG_HD void feed(const uint8_t *p, uint32_t n)
    {
        for (uint32_t k = 0; k < n; k++)
            feed(p[k]);
    }
    RG_HD bool done() const { return ok && label != 0 && total <= 253u; }
};

/* dotted-quad IPv4: four parts of 1-3 digits, each at most 255, no leading zero */
RG_HD bool rv_ipv4_ok(const uint8_t *p, uint32_t n)
{
    uint32_t dots = 0, digits = 0, v = 0;
    bool ok = n != 0 && n <= 15u;
    for (uint32_t k = 0; k < n && ok; k++) {
        const uint8_t c = p[k];
        if (c == '.') {
            ok = digits != 0;
            dots++;
            digits = v = 0;
        } else if (c >= '0' && c <= '9') {
            ok = !(digits == 1u && v == 0u);
            v = v * 10u + (uint32_t)(c - '0');
            digits++;
            ok = ok && digits <= 3u && v <= 255u;
        } else {
            ok = false;
        }
    }
    return ok && digits != 0 && dots == 3u;
}

/* regk_decode reports an absent ttl as INT32_MIN, which is also what "ttl":-2147483648 reads as: only then is the
   member looked for (an unescaped `"ttl":-` can only be the member, a string's quotes are escaped) */
RG_HD bool rv_ttl_present(const Decoded &d, const uint8_t *json, uint32_t jn)
{
    if (d.ttl != INT32_MIN)
        return true;
    for (uint32_t k = 0; k + 7u <= jn; k++)
        if (rv_eq(json + k, 7u, "\"ttl\":-"))
            return true;
    return false;
}

struct RvNode {
    uint8_t cls, roles;
    int32_t ttl;                                /* a_ttl of a host record, srv_ttl of a service record */
};

/* Decoded.flags bits above the public REGK_DEC_* (internal, never returned by regk_decode): REGK_RESOLVE_ANY_FORM's
   general reader (regk_resolve_any.cuh) read the node, and found a ttl in it */
enum : uint32_t { RV_DEC_ANY_READ = 1u << 16, RV_DEC_TTL_IN = 1u << 17 };

/* Node j from its regk_decode record (host_nodes = 0), its data, its domain and its ports: the first failing rule of
   include/regk.h REGK_RSV_* decides the class.  ANY: a node the general reader read says itself whether it has a ttl. */
template <bool ANY = false>
RG_HD RvNode rv_classify(const Decoded &d, const uint8_t *json, uint32_t jn, const uint8_t *dom, const uint32_t *ports,
    int32_t dflt_host, int32_t dflt_srv)
{
    RvNode r;
    r.cls = RV_OK;
    r.roles = 0;
    r.ttl = 0;
    const uint32_t bad = DEC_NOT_CANONICAL | DEC_KEY_MISMATCH | DEC_ADDR_MISMATCH | DEC_BAD_NUMBER | DEC_BAD_PATH;
    const bool host = (d.flags & DEC_HOST_RECORD) != 0, svc = (d.flags & DEC_SERVICE_RECORD) != 0;
    if (jn == 0) {
        r.cls = RV_EMPTY;
        return r;
    }
    if ((d.flags & bad) || !(d.flags & DEC_PATH_OK) || !(host || svc)) {
        r.cls = RV_NOT_RECORD;
        return r;
    }
    RvName nm;
    nm.init();
    nm.feed(dom, d.dom_len);
    bool name_ok = nm.done();
    if (svc) {                                  /* the SRV owner <srvce>.<proto>.<name> */
        RvName o;
        o.init();
        o.feed(json + d.type_pos, d.type_len);
        o.feed('.');
        o.feed(json + d.addr_pos, d.addr_len);
        o.feed('.');
        o.feed(dom, d.dom_len);
        name_ok = name_ok && o.done();
    }
    const uint32_t tr = host ? rv_type_roles(json + d.type_pos, d.type_len) : 0u;
    const bool ttl_in = (ANY && (d.flags & RV_DEC_ANY_READ)) ? (d.flags & RV_DEC_TTL_IN) != 0 : rv_ttl_present(d, json, jn);
    const uint32_t np = svc ? 1u : (d.nports == 0xFFFFFFFFu ? 0u : d.nports);
    uint32_t maxport = 0;
    for (uint32_t k = 0; k < np; k++)
        maxport = ports[k] > maxport ? ports[k] : maxport;
    r.cls = !name_ok ? RV_BAD_NAME : (host && !tr) ? RV_UNKNOWN_TYPE : (host && !rv_ipv4_ok(json + d.addr_pos, d.addr_len)) ?
        RV_BAD_ADDRESS : (ttl_in && d.ttl < 0) ? RV_BAD_TTL : maxport > 65535u ? RV_BAD_PORT : RV_OK;
    r.ttl = ttl_in ? d.ttl : (host ? dflt_host : dflt_srv);
    if (r.cls == RV_OK)
        r.roles = svc ? RV_ROLE_SERVICE : (uint8_t)(((tr & 1u) ? RV_ROLE_HOST_A : 0) | ((tr & 2u) ? RV_ROLE_CHILD : 0));
    return r;
}

/* "<name>.\t<ttl>\tIN\tA\t<addr>\n" */
RG_HD uint64_t rv_a_len(uint32_t name, int32_t ttl, uint32_t addr)
{
    return (uint64_t)name + addr + ndigits_i32(ttl) + 9u;
}

/* "<srvce>.<proto>.<service>.\t<ttl>\tIN\tSRV\t0 10 <port> <child>.\n" */
RG_HD uint64_t rv_srv_len(uint32_t srvce, uint32_t proto, uint32_t service, int32_t ttl, uint32_t port, uint32_t child)
{
    return (uint64_t)srvce + proto + service + child + ndigits_i32(ttl) + ndigits_u32(port) + 20u;
}

RG_HD uint8_t *rv_put(uint8_t *o, const uint8_t *s, uint32_t n)
{
    for (uint32_t k = 0; k < n; k++)
        o[k] = s[k];
    return o + n;
}

RG_HD uint8_t *rv_put_dec(uint8_t *o, uint32_t v)
{
    const uint32_t n = ndigits_u32(v);
    for (uint32_t k = n; k > 0; k--) {
        o[k - 1] = (uint8_t)('0' + v % 10u);
        v /= 10u;
    }
    return o + n;
}

RG_HD uint8_t *rv_put_a(uint8_t *o, const uint8_t *name, uint32_t nl, int32_t ttl, const uint8_t *addr, uint32_t al)
{
    o = rv_put(o, name, nl);
    *o++ = '.';
    *o++ = '\t';
    o = rv_put_dec(o, (uint32_t)ttl);
    *o++ = '\t';
    *o++ = 'I';
    *o++ = 'N';
    *o++ = '\t';
    *o++ = 'A';
    *o++ = '\t';
    o = rv_put(o, addr, al);
    *o++ = '\n';
    return o;
}

RG_HD uint8_t *rv_put_srv(uint8_t *o, const uint8_t *srvce, uint32_t sl, const uint8_t *proto, uint32_t pl, const uint8_t *service,
    uint32_t nl, int32_t ttl, uint32_t port, const uint8_t *child, uint32_t cl)
{
    o = rv_put(o, srvce, sl);
    *o++ = '.';
    o = rv_put(o, proto, pl);
    *o++ = '.';
    o = rv_put(o, service, nl);
    *o++ = '.';
    *o++ = '\t';
    o = rv_put_dec(o, (uint32_t)ttl);
    *o++ = '\t';
    *o++ = 'I';
    *o++ = 'N';
    *o++ = '\t';
    *o++ = 'S';
    *o++ = 'R';
    *o++ = 'V';
    *o++ = '\t';
    *o++ = '0';
    *o++ = ' ';
    *o++ = '1';
    *o++ = '0';
    *o++ = ' ';
    o = rv_put_dec(o, port);
    *o++ = ' ';
    o = rv_put(o, child, cl);
    *o++ = '.';
    *o++ = '\n';
    return o;
}

}  /* namespace regk */

#if defined(__CUDACC__)
#include "regk_kernels.cuh"

namespace regk {

constexpr uint32_t RV_TILE = 128;               /* items per CTA of the scanned passes */
/* counters[]: [0] smallest node with bad offsets (regk_reconcile_insert_kernel's RC_C_BAD), [1] smallest node with an
   earlier node's path (both ~0 = none), then the totals the host reads */
enum { RV_C_BAD = 0, RV_C_DUP = 1, RV_C_ANSWERS = 2, RV_C_ADDITIONAL = 3, RV_C_QUERIES = 4, RV_C_TEXT = 5, RV_C_UNRESOLVED = 6,
       RV_NCOUNTERS = 8 };

struct ResolveParams {
    uint64_t m;
    const uint8_t *path;
    const unsigned long long *path_off;         /* [m + 1] */
    const uint8_t *json;
    const unsigned long long *json_off;
    uint64_t path_total;                        /* readable bytes of the path stream */
    const Decoded *dec;                         /* regk_decode_kernel's records, domains (slot layout) and ports */
    const uint8_t *dom;
    const uint32_t *ports;
    int32_t dflt_host, dflt_srv;
    uint32_t mask;                              /* the insert pass's table: slots - 1, node + 1 per slot */
    const uint32_t *table;
    const uint32_t *slot;                       /* [m] node j's slot */
    uint8_t *cls, *roles;                       /* [m] */
    int32_t *ttl;                               /* [m] */
    uint32_t *key, *val;                        /* [m] sort input: the service of node j (m: none), j */
    const uint32_t *skey, *sval;                /* [m] sorted */
    uint32_t *first, *end;                      /* [m] service s: its children at sorted positions [first, end) */
    unsigned long long *cum[3];                 /* [m + 1] A / SRV / additional bytes per sorted position, then their
                                                   exclusive prefixes */
    unsigned long long *ctile[3], *csuper[3];   /* two-level totals of cum */
    unsigned long long *ntile[3], *nsuper[3];   /* ... of the per-node queries, section bytes, unresolved flags */
    unsigned long long *node_q;                 /* [m] node j's first query */
    uint8_t *q_kind;
    unsigned long long *q_node, *sec_off, *unresolved;
    unsigned long long *counters;
    uint8_t *text;
};

/* exclusive prefix inside the CTA of K values per thread, and the CTA's totals (once per kernel: static shared) */
template <int K>
__device__ __forceinline__ void rv_block_scan(unsigned long long (&v)[K], unsigned long long (&tot)[K])
{
    __shared__ unsigned long long s_w[K][RV_TILE / 32];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    #pragma unroll
    for (int k = 0; k < K; k++) {
        unsigned long long x = v[k];
        #pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const unsigned long long y = __shfl_up_sync(0xFFFFFFFFu, x, d);
            if (lane >= (uint32_t)d)
                x += y;
        }
        if (lane == 31)
            s_w[k][warp] = x;
        v[k] = x - v[k];
    }
    __syncthreads();
    #pragma unroll
    for (int k = 0; k < K; k++) {
        unsigned long long b = 0, t = 0;
        #pragma unroll
        for (uint32_t w = 0; w < RV_TILE / 32; w++) {
            b += w < warp ? s_w[k][w] : 0ull;
            t += s_w[k][w];
        }
        v[k] += b;
        tot[k] = t;
    }
}

__device__ __forceinline__ void rv_add_total(unsigned long long *tile_total, unsigned long long *super_total, uint32_t tile,
    unsigned long long v)
{
    tile_total[tile] = v;
    if (v)
        atomicAdd(super_total + tile / SUPER, v);
}

/* the exclusive base of `tile` (warp 0, every lane gets it): the project's two-level totals with 64-bit tile totals */
__device__ __forceinline__ unsigned long long rv_tile_base(const unsigned long long *tile_total, const unsigned long long *super_total,
    uint32_t tile)
{
    const uint32_t lane = threadIdx.x & 31u, nsuper = tile / SUPER;
    unsigned long long acc = 0;
    for (uint32_t i = lane; i < nsuper; i += 32)
        acc += super_total[i];
    for (uint32_t i = nsuper * SUPER + lane; i < tile; i += 32)
        acc += tile_total[i];
    #pragma unroll
    for (int d = 16; d > 0; d >>= 1)
        acc += __shfl_xor_sync(0xFFFFFFFFu, acc, d);
    return acc;
}

template <int K>
__device__ __forceinline__ void rv_tile_bases(unsigned long long *const (&tile_total)[3], unsigned long long *const (&super_total)[3],
    uint32_t tile, unsigned long long (&base)[K])
{
    __shared__ unsigned long long s_base[K];
    if (threadIdx.x < 32) {
        #pragma unroll
        for (int k = 0; k < K; k++) {
            const unsigned long long b = rv_tile_base(tile_total[k], super_total[k], tile);
            if (threadIdx.x == 0)
                s_base[k] = b;
        }
    }
    __syncthreads();
    #pragma unroll
    for (int k = 0; k < K; k++)
        base[k] = s_base[k];
}

/* ---- classify: duplicate path, class, roles, TTL (ANY: regk_resolve_any.cuh's variant) ---- */
template <bool ANY>
__device__ __forceinline__ void rv_classify_node(const ResolveParams &p)
{
    const uint64_t j = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (j >= p.m)
        return;
    if (p.table[p.slot[j]] != (uint32_t)j + 1u)
        atomicMin(p.counters + RV_C_DUP, (unsigned long long)j);
    const unsigned long long q0 = p.json_off[j];
    const Decoded d = p.dec[j];
    const RvNode r = rv_classify<ANY>(d, p.json + q0, (uint32_t)(p.json_off[j + 1] - q0), p.dom + p.path_off[j],
        p.ports + (q0 >> 1), p.dflt_host, p.dflt_srv);
    p.cls[j] = r.cls;
    p.roles[j] = r.roles;
    p.ttl[j] = r.ttl;
}

__global__ void __launch_bounds__(256) regk_resolve_classify_kernel(const ResolveParams p)
{
    rv_classify_node<false>(p);
}

/* ---- join: the service node each candidate child belongs to ---- */
__global__ void __launch_bounds__(256) regk_resolve_join_kernel(const ResolveParams p)
{
    const uint64_t j = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (j >= p.m)
        return;
    uint32_t key = (uint32_t)p.m;
    if (p.roles[j] & RV_ROLE_CHILD) {
        const unsigned long long o0 = p.path_off[j];
        uint32_t q = (uint32_t)(p.path_off[j + 1] - o0);
        while (q > 0 && p.path[o0 + q - 1] != '/')
            q--;
        const uint32_t plen = q > 1 ? q - 1 : 0;                /* dirname; "/" is never a service record */
        if (plen) {
            const uint32_t *W = reinterpret_cast<const uint32_t *>(p.path);
            uint32_t slot = string_hash32_clamped(W, o0, plen, p.path_total) & p.mask;
            for (;;) {
                const uint32_t cur = p.table[slot];
                if (cur == 0u)
                    break;
                const uint64_t k = cur - 1u;
                const unsigned long long k0 = p.path_off[k];
                if ((uint32_t)(p.path_off[k + 1] - k0) == plen && string_equal2(W, o0, p.path_total, W, k0, p.path_total, plen)) {
                    if (p.cls[k] == RV_OK && (p.roles[k] & RV_ROLE_SERVICE))
                        key = (uint32_t)k;
                    break;
                }
                slot = (slot + 1u) & p.mask;
            }
        }
    }
    p.key[j] = key;
    p.val[j] = (uint32_t)j;
}

/* the bytes of child c's lines under service s: its A answer, its SRV answers (*nsrv lines), its additional */
__device__ __forceinline__ void rv_child_bytes(const ResolveParams &p, uint32_t s, uint32_t c, unsigned long long (&b)[3], uint32_t *nsrv)
{
    const Decoded &ds = p.dec[s], &dc = p.dec[c];
    const int32_t ts = p.ttl[s], tc = p.ttl[c];
    b[0] = rv_a_len(ds.dom_len, min(ts, tc), dc.addr_len);
    const bool own = dc.nports != 0xFFFFFFFFu;
    const uint32_t np = own ? dc.nports : 1u;
    const uint32_t *pp = own ? p.ports + (p.json_off[c] >> 1) : p.ports + (p.json_off[s] >> 1);
    unsigned long long srv = 0;
    for (uint32_t k = 0; k < np; k++)
        srv += rv_srv_len(ds.type_len, ds.addr_len, ds.dom_len, ts, pp[k], dc.dom_len);
    b[1] = srv;
    b[2] = np ? rv_a_len(dc.dom_len, tc, dc.addr_len) : 0ull;
    *nsrv = np;
}

/* ---- child_len: per sorted position, the child's three byte counts; each service's range ---- */
__global__ void __launch_bounds__(RV_TILE) regk_resolve_child_len_kernel(const ResolveParams p)
{
    const uint64_t i = (uint64_t)blockIdx.x * RV_TILE + threadIdx.x;
    unsigned long long b[3] = {0ull, 0ull, 0ull}, tot[3];
    uint32_t lines = 0, adds = 0;
    if (i < p.m) {
        const uint32_t s = p.skey[i];
        if (s < p.m) {
            uint32_t nsrv = 0;
            rv_child_bytes(p, s, p.sval[i], b, &nsrv);
            lines = 1u + nsrv;
            adds = nsrv ? 1u : 0u;
            if (i == 0 || p.skey[i - 1] != s)
                p.first[s] = (uint32_t)i;
            if (i + 1 == p.m || p.skey[i + 1] != s)
                p.end[s] = (uint32_t)i + 1u;
        }
        #pragma unroll
        for (int k = 0; k < 3; k++)
            p.cum[k][i] = b[k];
    }
    #pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        lines += __shfl_xor_sync(0xFFFFFFFFu, lines, d);
        adds += __shfl_xor_sync(0xFFFFFFFFu, adds, d);
    }
    if ((threadIdx.x & 31u) == 0 && lines) {
        atomicAdd(p.counters + RV_C_ANSWERS, (unsigned long long)lines);
        atomicAdd(p.counters + RV_C_ADDITIONAL, (unsigned long long)adds);
    }
    rv_block_scan<3>(b, tot);
    if (threadIdx.x == 0) {
        #pragma unroll
        for (int k = 0; k < 3; k++)
            rv_add_total(p.ctile[k], p.csuper[k], blockIdx.x, tot[k]);
    }
}

/* ---- child_scan: the byte counts become exclusive prefixes over the sorted positions; cum[k][m] = the total ---- */
__global__ void __launch_bounds__(RV_TILE) regk_resolve_child_scan_kernel(const ResolveParams p)
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

/* node j's queries and its sections' bytes: A answers, SRV answers, SRV additionals (a HOST_A node: sec[0] only) */
__device__ __forceinline__ uint32_t rv_node_sections(const ResolveParams &p, uint64_t j, unsigned long long (&sec)[3])
{
    const uint8_t r = p.roles[j];
    sec[0] = sec[1] = sec[2] = 0ull;
    if (r & RV_ROLE_HOST_A) {
        const Decoded &d = p.dec[j];
        sec[0] = rv_a_len(d.dom_len, p.ttl[j], d.addr_len);
        return 1u;
    }
    if (r & RV_ROLE_SERVICE) {
        const uint32_t f = p.first[j], e = p.end[j];
        #pragma unroll
        for (int k = 0; k < 3; k++)
            sec[k] = p.cum[k][e] - p.cum[k][f];
        return 2u;
    }
    return 0u;
}

/* ---- qlen: per-tile totals of queries, section bytes and unresolved nodes ---- */
__global__ void __launch_bounds__(RV_TILE) regk_resolve_qlen_kernel(const ResolveParams p)
{
    const uint64_t j = (uint64_t)blockIdx.x * RV_TILE + threadIdx.x;
    unsigned long long v[4] = {0ull, 0ull, 0ull, 0ull}, tot[4];
    if (j < p.m) {
        unsigned long long sec[3];
        const uint32_t nq = rv_node_sections(p, j, sec);
        v[0] = nq;
        v[1] = sec[0] + sec[1] + sec[2];
        v[2] = p.cls[j] >= RV_NOT_RECORD ? 1ull : 0ull;
        v[3] = nq == 1u ? 1ull : 0ull;                          /* a HOST_A answer line */
    }
    rv_block_scan<4>(v, tot);
    if (threadIdx.x == 0) {
        #pragma unroll
        for (int k = 0; k < 3; k++)
            rv_add_total(p.ntile[k], p.nsuper[k], blockIdx.x, tot[k]);
        if (tot[3])
            atomicAdd(p.counters + RV_C_ANSWERS, tot[3]);
    }
}

/* ---- place: q_kind, q_node, sec_off, node_q, the unresolved list and the totals ---- */
__global__ void __launch_bounds__(RV_TILE) regk_resolve_place_kernel(const ResolveParams p)
{
    const uint64_t j = (uint64_t)blockIdx.x * RV_TILE + threadIdx.x;
    unsigned long long base[3], v[3] = {0ull, 0ull, 0ull}, tot[3], sec[3] = {0ull, 0ull, 0ull};
    rv_tile_bases<3>(p.ntile, p.nsuper, blockIdx.x, base);
    uint32_t nq = 0;
    bool unres = false;
    if (j < p.m) {
        nq = rv_node_sections(p, j, sec);
        unres = p.cls[j] >= RV_NOT_RECORD;
        v[0] = nq;
        v[1] = sec[0] + sec[1] + sec[2];
        v[2] = unres ? 1ull : 0ull;
    }
    const unsigned long long own1 = v[1];
    rv_block_scan<3>(v, tot);
    if (j >= p.m)
        return;
    const unsigned long long q = base[0] + v[0], off = base[1] + v[1];
    if (nq) {
        p.node_q[j] = q;
        p.q_kind[q] = nq == 1u ? RV_Q_HOST_A : RV_Q_SERVICE_A;
        p.q_node[q] = j;
        p.sec_off[2 * q] = off;
        p.sec_off[2 * q + 1] = off + sec[0];
    }
    if (nq == 2u) {
        p.q_kind[q + 1] = RV_Q_SERVICE_SRV;
        p.q_node[q + 1] = j;
        p.sec_off[2 * q + 2] = off + sec[0];
        p.sec_off[2 * q + 3] = off + sec[0] + sec[1];
    }
    if (unres)
        p.unresolved[base[2] + v[2]] = j;
    if (j + 1 == p.m) {
        p.sec_off[2 * (q + nq)] = off + own1;
        p.counters[RV_C_QUERIES] = q + nq;
        p.counters[RV_C_TEXT] = off + own1;
        p.counters[RV_C_UNRESOLVED] = base[2] + v[2] + (unres ? 1ull : 0ull);
    }
}

/* ---- emit: one thread per HOST_A node (first m threads), one per child (sorted positions) ---- */
__global__ void __launch_bounds__(256) regk_resolve_emit_kernel(const ResolveParams p)
{
    const uint64_t t = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (t < p.m) {
        if (!(p.roles[t] & RV_ROLE_HOST_A))
            return;
        const Decoded &d = p.dec[t];
        rv_put_a(p.text + p.sec_off[2 * p.node_q[t]], p.dom + p.path_off[t], d.dom_len, p.ttl[t], p.json + p.json_off[t] + d.addr_pos,
            d.addr_len);
        return;
    }
    const uint64_t i = t - p.m;
    if (i >= p.m)
        return;
    const uint32_t s = p.skey[i];
    if (s >= p.m)
        return;
    const uint32_t c = p.sval[i], f = p.first[s];
    const unsigned long long qa = p.node_q[s];
    const Decoded &ds = p.dec[s], &dc = p.dec[c];
    const int32_t ts = p.ttl[s], tc = p.ttl[c];
    const uint8_t *sname = p.dom + p.path_off[s], *cname = p.dom + p.path_off[c];
    const uint8_t *caddr = p.json + p.json_off[c] + dc.addr_pos;
    rv_put_a(p.text + p.sec_off[2 * qa] + (p.cum[0][i] - p.cum[0][f]), sname, ds.dom_len, min(ts, tc), caddr, dc.addr_len);
    const bool own = dc.nports != 0xFFFFFFFFu;
    const uint32_t np = own ? dc.nports : 1u;
    const uint32_t *pp = own ? p.ports + (p.json_off[c] >> 1) : p.ports + (p.json_off[s] >> 1);
    const uint8_t *sj = p.json + p.json_off[s];
    uint8_t *o = p.text + p.sec_off[2 * qa + 2] + (p.cum[1][i] - p.cum[1][f]);
    for (uint32_t k = 0; k < np; k++)
        o = rv_put_srv(o, sj + ds.type_pos, ds.type_len, sj + ds.addr_pos, ds.addr_len, sname, ds.dom_len, ts, pp[k], cname, dc.dom_len);
    if (np)
        rv_put_a(p.text + p.sec_off[2 * qa + 3] + (p.cum[2][i] - p.cum[2][f]), cname, dc.dom_len, tc, caddr, dc.addr_len);
}

}  /* namespace regk */
#endif /* __CUDACC__ */
#endif /* REGK_RESOLVE_CUH */
