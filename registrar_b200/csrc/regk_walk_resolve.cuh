/*
 * regk_walk_resolve.cuh — re-resolve a walk's snapshot incrementally (regk_walk_resolve): regk_resolve's metadata
 * passes run unchanged, and the text is assembled from the last call's text wherever a line's inputs did not change.
 *
 * identity  one word per snapshot node: its index at the last successful regk_walk_resolve, or WR_NONE.  Appended
 *           nodes get WR_NONE; the keep pass compacts the words alongside regk_walk_keep_kernel (its tile totals, its
 *           predicate) and clears the identity of a node whose refresh-level getData brought data bytes that differ
 *           from its old ones, so the word moves with its node through a rebuild.
 * pieces    the text in order is, per node ascending: a HOST_A node's section; a service's child A lines, then its
 *           children's SRV runs, then their additional lines (each in sorted child order).  Piece slot of HOST_A node j:
 *           j + 3 lb(j), lb(j) = the sorted child positions whose service is below j; child position i of service s
 *           (positions [f, e), n = e - f): s + 3 f + 1 + (i - f) + k n for its run k = A, SRV, additional.  Slots are
 *           dense in text order; a slot no piece lands on is empty.
 *   plan    one thread per HOST_A node and per sorted child position: each piece's kind (copy from the old text or
 *           fresh), length and destination from the new sec_off / cum, and a copy's source from the old run offsets.
 *           A HOST_A section is copied when its node has an identity; a child's runs when the child and its service
 *           both have one.
 *   seg     per slot (two-level totals, block scan): a nonempty piece starts a segment unless the slot before holds a
 *           piece of the same kind whose source ends where this one's starts (fresh pieces are laid out in the scratch
 *           stream in slot order) and whose destination lies in the same 2^WR_WINDOW-byte window of the text, so a
 *           segment stays short: the gather's CTAs then get even work, and a segment is far below 2^32 bytes.  Segment k's source, select and destination; a fresh piece's scratch offset replaces its source.
 *   fresh   the formatted pieces into the scratch stream, by rv_put_a / rv_put_srv.
 *   gather  regk_mkdirp_len_kernel and regk_walk_rebuild_kernel over the segments (source 0: the old text, 1: scratch).
 *   stamp   per node, where its HOST_A section and its three child runs start in this call's text, and identity = j.
 */
#ifndef REGK_WALK_RESOLVE_CUH
#define REGK_WALK_RESOLVE_CUH

#include "regk_resolve.cuh"
#include "regk_walk_watch.cuh"

namespace regk {

constexpr uint32_t WR_NONE = 0xFFFFFFFFu;
enum : uint8_t { WR_EMPTY = 0, WR_COPY = 1, WR_FRESH = 2 };
enum { WR_C_FRESH_NODES = 0, WR_NCOUNTERS = 2 };
constexpr uint32_t WR_WINDOW = 8;               /* a segment's pieces start in one 256-byte window of the text */

/* ---- keep identity: regk_walk_keep_kernel's compaction of the identities; a replaced node keeps its identity only
   when its new data bytes equal its old ones ---- */
__global__ void __launch_bounds__(RP_TILE) regk_walk_keep_ident_kernel(const WalkKeepParams p, const uint32_t *ident,
    uint32_t *nident, const uint8_t *old_data, const uint8_t *ds)
{
    __shared__ uint32_t s_warp[WARPS];
    __shared__ unsigned long long s_base;
    if (threadIdx.x < 32) {
        const unsigned long long base = tile_base_from_totals(p.tile_total, p.super_total, blockIdx.x);
        if (threadIdx.x == 0)
            s_base = base;
    }
    const uint64_t j = (uint64_t)blockIdx.x * RP_TILE + threadIdx.x;
    const uint32_t mk = j < p.m ? p.mark[j] : WK_REMOVED;
    const bool keep = !(mk & WK_REMOVED);
    uint32_t tot;
    const uint32_t r = block_scan<uint32_t>(s_warp, keep ? 1u : 0u, &tot);     /* its barriers publish s_base */
    if (!keep)
        return;
    uint32_t id = ident[j];
    if (id != WR_NONE && (mk & WK_REPLACED)) {
        const unsigned long long o0 = p.json_off[j];
        const uint32_t n = (uint32_t)(p.json_off[j + 1] - o0);
        bool same = n == p.rlen[j];
        const uint8_t *a = old_data + o0, *b = ds + p.rpos[j];
        for (uint32_t k = 0; same && k < n; k++)
            same = a[k] == b[k];
        id = same ? id : WR_NONE;
    }
    nident[s_base + r] = id;
}

struct WalkResolveParams {
    ResolveParams r;                            /* the resolve's arrays, as its passes left them */
    const uint32_t *ident;                      /* [m] identity per node */
    const unsigned long long *run_old;          /* [4 m_old] the last call's HOST_A section / child run starts */
    unsigned long long *run_new;                /* [4 m] this call's */
    uint32_t *ident_out;                        /* stamp: [m] */
    uint64_t n_slots;
    uint8_t *kind;                              /* [n_slots] WR_* */
    uint32_t *len;
    unsigned long long *src, *dest;             /* a copy's old-text offset (a fresh piece's scratch offset after seg) */
    unsigned long long *stile[2], *ssuper[2];   /* two-level totals: segment starts, fresh bytes */
    unsigned long long *seg_src, *seg_dest;     /* [segments] */
    uint8_t *seg_sel;
    uint32_t *seg_len;
    uint64_t n_seg, text_total;
    uint8_t *scratch;
    unsigned long long *counters;               /* [WR_NCOUNTERS] */
};

/* the sorted child positions whose service is below j */
__device__ __forceinline__ uint64_t wr_lower(const ResolveParams &p, uint64_t j)
{
    uint64_t lo = 0, hi = p.m;
    while (lo < hi) {
        const uint64_t mid = (lo + hi) >> 1;
        if (p.skey[mid] < j)
            lo = mid + 1;
        else
            hi = mid;
    }
    return lo;
}

/* the section start of run k (0 A, 1 SRV, 2 additional) of service s's query qa */
__device__ __forceinline__ unsigned long long wr_run_base(const ResolveParams &p, unsigned long long qa, int k)
{
    return p.sec_off[2 * qa + (k == 0 ? 0 : k + 1)];
}

__device__ __forceinline__ void wr_piece(const WalkResolveParams &w, uint64_t slot, unsigned long long dest, unsigned long long n,
    bool copy, unsigned long long src)
{
    w.kind[slot] = n ? (copy ? WR_COPY : WR_FRESH) : WR_EMPTY;
    w.len[slot] = (uint32_t)n;
    w.src[slot] = copy ? src : 0ull;
    w.dest[slot] = dest;
}

/* ---- plan: one thread per HOST_A node (first m threads), one per sorted child position ---- */
__global__ void __launch_bounds__(256) regk_walk_resolve_plan_kernel(const WalkResolveParams w)
{
    const ResolveParams &p = w.r;
    const uint64_t t = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    const bool fresh_node = t < p.m && w.ident[t] == WR_NONE;
    const uint32_t nf = __popc(__ballot_sync(0xFFFFFFFFu, fresh_node));
    if ((threadIdx.x & 31u) == 0 && nf)
        atomicAdd(w.counters + WR_C_FRESH_NODES, (unsigned long long)nf);
    if (t < p.m) {
        if (!(p.roles[t] & RV_ROLE_HOST_A))
            return;
        const unsigned long long q = p.node_q[t], d = p.sec_off[2 * q];
        const uint32_t id = w.ident[t];
        wr_piece(w, t + 3 * wr_lower(p, t), d, p.sec_off[2 * q + 2] - d, id != WR_NONE, id != WR_NONE ? w.run_old[4ull * id] : 0ull);
        return;
    }
    const uint64_t i = t - p.m;
    if (i >= p.m)
        return;
    const uint32_t s = p.skey[i];
    if (s >= p.m)
        return;
    const uint32_t c = p.sval[i], f = p.first[s], n = p.end[s] - f;
    const uint32_t ic = w.ident[c];
    const bool copy = ic != WR_NONE && w.ident[s] != WR_NONE;
    const unsigned long long qa = p.node_q[s];
    const uint64_t slot = (uint64_t)s + 3ull * f + 1ull + (i - f);
    #pragma unroll
    for (int k = 0; k < 3; k++) {
        const unsigned long long d = wr_run_base(p, qa, k) + (p.cum[k][i] - p.cum[k][f]);
        wr_piece(w, slot + (uint64_t)k * n, d, p.cum[k][i + 1] - p.cum[k][i], copy, copy ? w.run_old[4ull * ic + 1 + k] : 0ull);
    }
}

/* slot r starts a segment: a nonempty piece that does not continue the piece of slot r - 1 */
__device__ __forceinline__ bool wr_starts(const WalkResolveParams &w, uint64_t r, uint8_t kd)
{
    if (kd == WR_EMPTY)
        return false;
    if (r == 0 || w.kind[r - 1] != kd || (w.dest[r - 1] >> WR_WINDOW) != (w.dest[r] >> WR_WINDOW))
        return true;
    return kd == WR_COPY && w.src[r - 1] + w.len[r - 1] != w.src[r];
}

/* segment starts and fresh bytes of slot r as one scan value, count << 40 | bytes (a CTA's bytes stay below 2^40) */
__device__ __forceinline__ unsigned long long wr_seg_value(const WalkResolveParams &w, uint64_t r, uint8_t *kd, bool *st)
{
    *kd = r < w.n_slots ? w.kind[r] : WR_EMPTY;
    *st = r < w.n_slots && wr_starts(w, r, *kd);
    return (*st ? 1ull << 40 : 0ull) | (*kd == WR_FRESH ? (unsigned long long)w.len[r] : 0ull);
}

/* ---- seg count: per-tile totals of segment starts and fresh bytes ---- */
__global__ void __launch_bounds__(RV_TILE) regk_walk_resolve_seg_count_kernel(const WalkResolveParams w)
{
    __shared__ unsigned long long s_warp[RV_TILE / 32];
    const uint64_t r = (uint64_t)blockIdx.x * RV_TILE + threadIdx.x;
    uint8_t kd;
    bool st;
    const unsigned long long v = wr_seg_value(w, r, &kd, &st);
    unsigned long long tot;
    block_scan<unsigned long long>(s_warp, v, &tot);
    if (threadIdx.x == 0) {
        rv_add_total(w.stile[0], w.ssuper[0], blockIdx.x, tot >> 40);
        rv_add_total(w.stile[1], w.ssuper[1], blockIdx.x, tot & ((1ull << 40) - 1));
    }
}

/* ---- seg: segment k's source, select and destination; a fresh piece's scratch offset ---- */
__global__ void __launch_bounds__(RV_TILE) regk_walk_resolve_seg_kernel(const WalkResolveParams w)
{
    __shared__ unsigned long long s_warp[RV_TILE / 32];
    __shared__ unsigned long long s_base[2];
    if (threadIdx.x < 32) {
        #pragma unroll
        for (int k = 0; k < 2; k++) {
            const unsigned long long b = rv_tile_base(w.stile[k], w.ssuper[k], blockIdx.x);
            if (threadIdx.x == 0)
                s_base[k] = b;
        }
    }
    const uint64_t r = (uint64_t)blockIdx.x * RV_TILE + threadIdx.x;
    uint8_t kd;
    bool st;
    const unsigned long long v = wr_seg_value(w, r, &kd, &st);
    unsigned long long tot;
    const unsigned long long x = block_scan<unsigned long long>(s_warp, v, &tot);   /* its barriers publish s_base */
    if (kd == WR_EMPTY)
        return;
    const unsigned long long sc = s_base[1] + (x & ((1ull << 40) - 1));
    if (kd == WR_FRESH)
        w.src[r] = sc;
    if (st) {
        const unsigned long long k = s_base[0] + (x >> 40);
        w.seg_sel[k] = kd == WR_FRESH ? 1u : 0u;
        w.seg_src[k] = kd == WR_FRESH ? sc : w.src[r];
        w.seg_dest[k] = w.dest[r];
    }
}

/* ---- seg len: segment k ends where segment k + 1 (or the text) starts ---- */
__global__ void __launch_bounds__(256) regk_walk_resolve_seg_len_kernel(const WalkResolveParams w)
{
    const uint64_t k = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (k >= w.n_seg)
        return;
    const unsigned long long e = k + 1 < w.n_seg ? w.seg_dest[k + 1] : w.text_total;
    w.seg_len[k] = (uint32_t)(e - w.seg_dest[k]);
}

/* ---- fresh: the formatted pieces into the scratch stream (regk_resolve_emit_kernel's lines) ---- */
__global__ void __launch_bounds__(256) regk_walk_resolve_fresh_kernel(const WalkResolveParams w)
{
    const ResolveParams &p = w.r;
    const uint64_t t = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (t < p.m) {
        if (!(p.roles[t] & RV_ROLE_HOST_A) || w.ident[t] != WR_NONE)
            return;
        const Decoded &d = p.dec[t];
        rv_put_a(w.scratch + w.src[t + 3 * wr_lower(p, t)], p.dom + p.path_off[t], d.dom_len, p.ttl[t],
            p.json + p.json_off[t] + d.addr_pos, d.addr_len);
        return;
    }
    const uint64_t i = t - p.m;
    if (i >= p.m)
        return;
    const uint32_t s = p.skey[i];
    if (s >= p.m)
        return;
    const uint32_t c = p.sval[i], f = p.first[s], n = p.end[s] - f;
    if (w.ident[c] != WR_NONE && w.ident[s] != WR_NONE)
        return;
    const uint64_t slot = (uint64_t)s + 3ull * f + 1ull + (i - f);
    const Decoded &ds = p.dec[s], &dc = p.dec[c];
    const int32_t ts = p.ttl[s], tc = p.ttl[c];
    const uint8_t *sname = p.dom + p.path_off[s], *cname = p.dom + p.path_off[c];
    const uint8_t *caddr = p.json + p.json_off[c] + dc.addr_pos;
    rv_put_a(w.scratch + w.src[slot], sname, ds.dom_len, min(ts, tc), caddr, dc.addr_len);
    const bool own = dc.nports != 0xFFFFFFFFu;
    const uint32_t np = own ? dc.nports : 1u;
    if (!np)
        return;
    const uint32_t *pp = own ? p.ports + (p.json_off[c] >> 1) : p.ports + (p.json_off[s] >> 1);
    const uint8_t *sj = p.json + p.json_off[s];
    uint8_t *o = w.scratch + w.src[slot + n];
    for (uint32_t k = 0; k < np; k++)
        o = rv_put_srv(o, sj + ds.type_pos, ds.type_len, sj + ds.addr_pos, ds.addr_len, sname, ds.dom_len, ts, pp[k], cname, dc.dom_len);
    rv_put_a(w.scratch + w.src[slot + 2ull * n], cname, dc.dom_len, tc, caddr, dc.addr_len);
}

/* ---- stamp: where each node's HOST_A section and child runs start in this call's text; identity = j ---- */
__global__ void __launch_bounds__(256) regk_walk_resolve_stamp_kernel(const WalkResolveParams w)
{
    const ResolveParams &p = w.r;
    const uint64_t t = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (t < p.m) {
        w.ident_out[t] = (uint32_t)t;
        if (p.roles[t] & RV_ROLE_HOST_A)
            w.run_new[4 * t] = p.sec_off[2 * p.node_q[t]];
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
    #pragma unroll
    for (int k = 0; k < 3; k++)
        w.run_new[4ull * c + 1 + k] = wr_run_base(p, qa, k) + (p.cum[k][i] - p.cum[k][f]);
}

}  /* namespace regk */
#endif /* REGK_WALK_RESOLVE_CUH */
