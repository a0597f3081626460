/*
 * regk_walk_watch.cuh — keep a walked snapshot current with ZooKeeper watches (regk_walk_events, regk_walk_refresh and
 * the refresh level of regk_read_walk).
 *
 * marks     one word per snapshot node: WK_PENDING (its watch fired: re-read it), WK_REMOVED (NodeDeleted: drop it at
 *           the next rebuild), WK_REPLACED (only inside a refresh-level read: its getData reply replaces its data).
 * table     the snapshot's paths, node + 1 under the hash of its path (insert: nodes [j0, j1), so a table can be
 *           extended by the nodes a level appended; of two equal paths the smaller node keeps the slot, as in
 *           regk_replies_insert_kernel).  Built on demand, only after the snapshot changed.  Lookups compare byte for
 *           byte; a hash only picks a slot.
 * events    regk_events.cuh's cand and count passes and regk_replies.cuh's chain, unchanged; then
 *             map    one thread per chain frame: a notification's fields, the node its path names among the nodes not
 *                    marked removed, and for NodeDeleted the node at dirname(path), probed by hashing the path's prefix
 *                    in place.  Marks are only read, so every event of one call sees the snapshot as the call found it.
 *             mark   one thread per event: the marks ORed in, the pending / removed counts kept by each word's old value
 *                    (a removed node is never counted pending), so the result does not depend on the events' order.
 * rebuild   keep count / keep: the nodes not marked removed, compacted in order with their version, owner and mark
 *           (two-level totals, block scan); then regk_mkdirp_len_kernel's totals and the rebuild gather, output-
 *           stationary in whole 16-byte blocks as regk_mkdirp_gather_kernel, each node's bytes from one of two sources
 *           (the old snapshot, or the reply stream for a replaced node's data).
 * apply     a refresh-level read's getData replies onto their nodes: err 0 replaces version and owner in place and
 *           records where the data is, NONODE marks the node removed.
 * filter    a level's listed children whose path is not a snapshot node (optionally: not one left unmarked), compacted
 *           in listing order (filter count / filter), then packed as the next frontier by the mkdirp gather pair.
 * watch     the watch byte of every frame of a framing set to 1 (a frame's last byte), after regk_walk_frame_kernel.
 */
#ifndef REGK_WALK_WATCH_CUH
#define REGK_WALK_WATCH_CUH

#include "regk_events.cuh"
#include "regk_walk.cuh"

namespace regk {

enum : uint32_t { WK_PENDING = 1u, WK_REMOVED = 2u, WK_REPLACED = 4u };
enum { WM_PENDING = 0, WM_REMOVED, WM_NCOUNTERS };              /* the walk's persistent mark counts */

/* ---- watch: frame k's last byte (its watch flag) = 1 ---- */
__global__ void __launch_bounds__(256) regk_walk_watch_byte_kernel(uint8_t *out, const unsigned long long *out_off, uint64_t n)
{
    const uint64_t k = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (k < n)
        out[out_off[k + 1] - 1] = 1u;
}

/* ---- insert: nodes [j0, j1) into the path table ---- */
__global__ void __launch_bounds__(256) regk_walk_insert_kernel(uint32_t *table, uint32_t mask, const uint8_t *spath,
    const unsigned long long *soff, uint64_t j0, uint64_t j1)
{
    const uint64_t j = j0 + (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (j >= j1)
        return;
    const uint32_t *W = reinterpret_cast<const uint32_t *>(spath);
    const unsigned long long o = soff[j];
    const uint32_t len = (uint32_t)(soff[j + 1] - o);
    uint32_t slot = string_hash32(W, o, len) & mask;
    for (;;) {
        uint32_t cur = table[slot];
        if (cur == 0u) {
            cur = atomicCAS(table + slot, 0u, (uint32_t)j + 1u);
            if (cur == 0u)
                return;
        }
        const uint64_t k = cur - 1u;
        const unsigned long long k0 = soff[k];
        if ((uint32_t)(soff[k + 1] - k0) == len && string_equal(W, o, k0, len)) {
            if (cur > (uint32_t)j + 1u)
                atomicMin(table + slot, (uint32_t)j + 1u);
            return;
        }
        slot = (slot + 1u) & mask;
    }
}

/* the snapshot node whose path is the n bytes at o of V (readable below lim), or ~0 */
__device__ __forceinline__ uint64_t wk_find(const uint32_t *table, uint32_t mask, const uint8_t *spath,
    const unsigned long long *soff, const uint32_t *V, uint64_t o, uint64_t lim, uint32_t n)
{
    const uint32_t *W = reinterpret_cast<const uint32_t *>(spath);
    uint32_t slot = string_hash32_clamped(V, o, n, lim) & mask;
    for (;;) {
        const uint32_t cur = table[slot];
        if (cur == 0u)
            return ~0ull;
        const uint64_t j = cur - 1u;
        const unsigned long long j0 = soff[j];
        if ((uint32_t)(soff[j + 1] - j0) == n && string_equal2(W, j0, ~0ull, V, o, lim, n))
            return j;
        slot = (slot + 1u) & mask;
    }
}

/* ---- events: map (fields, node, parent) then mark ---- */
struct WalkEvParams {
    EvParams e;                                 /* r (the chain), tile_total / super_total (regk_events_count_kernel's), pos, type, state, zxid */
    const uint8_t *spath;                       /* the snapshot's paths (>= 16 bytes of slack) */
    const unsigned long long *soff;
    const uint32_t *table;
    uint32_t mask;
    uint32_t *mark;                             /* [m] */
    unsigned long long *node, *parent;          /* [events] */
    uint64_t n_ev;                              /* mark: the events */
    unsigned long long *mcount;                 /* [WM_NCOUNTERS] */
};

__global__ void __launch_bounds__(RP_TILE) regk_walk_events_kernel(const WalkEvParams wp)
{
    const EvParams &ep = wp.e;
    const RepParams &p = ep.r;
    __shared__ uint32_t s_warp[WARPS];
    __shared__ unsigned long long s_base;
    __shared__ uint32_t s_cnt[4];                   /* pings, replies, unmatched, other types */
    if (threadIdx.x < 4)
        s_cnt[threadIdx.x] = 0;
    if (threadIdx.x < 32) {
        const unsigned long long base = tile_base_from_totals(ep.tile_total, ep.super_total, blockIdx.x);
        if (threadIdx.x == 0)
            s_base = base;
    }
    const uint64_t c = (uint64_t)blockIdx.x * RP_TILE + threadIdx.x;
    const bool on = c < p.C && p.marked[c];
    const bool note = ev_is_note(p, c);
    uint32_t tot;
    const uint32_t r = block_scan<uint32_t>(s_warp, note ? 1u : 0u, &tot);      /* its barriers publish s_base, s_cnt */
    if (on && !note) {
        const int32_t xid = (int32_t)be32_at(p.s + p.cand[c] + 4);
        atomicAdd(&s_cnt[xid == -2 ? 0 : 1], 1u);
    } else if (note) {
        const uint64_t e = s_base + r;
        const unsigned long long pos = p.cand[c];
        const uint8_t *fr = p.s + pos;
        const int32_t type = (int32_t)be32_at(fr + 20);
        const uint32_t P = be32_at(fr + 28);
        const uint32_t *V = reinterpret_cast<const uint32_t *>(p.s);
        uint64_t j = ~0ull, par = ~0ull;
        if (type >= 2 && type <= 4) {
            j = wk_find(wp.table, wp.mask, wp.spath, wp.soff, V, pos + 32u, p.len, P);
            if (j != ~0ull && (wp.mark[j] & WK_REMOVED))
                j = ~0ull;
        }
        if (j != ~0ull && type == 2) {
            uint32_t d = P;                         /* dirname: up to the last '/', which is not the first byte */
            while (d > 0u && fr[32u + d - 1u] != '/')
                d--;
            if (d > 1u) {
                par = wk_find(wp.table, wp.mask, wp.spath, wp.soff, V, pos + 32u, p.len, d - 1u);
                if (par != ~0ull && (wp.mark[par] & WK_REMOVED))
                    par = ~0ull;
            }
        }
        if (j == ~0ull)
            atomicAdd(&s_cnt[2], 1u);
        if (type == -1 || type >= 5)
            atomicAdd(&s_cnt[3], 1u);
        ep.pos[e] = pos;
        ep.type[e] = type;
        ep.state[e] = (int32_t)be32_at(fr + 24);
        ep.zxid[e] = st_be64_at(fr + 8);
        wp.node[e] = j;
        wp.parent[e] = par;
    }
    if (c + 1 == p.C)
        p.counters[EQ_NEV] = s_base + tot;
    __syncthreads();
    if (threadIdx.x < 4 && s_cnt[threadIdx.x])
        atomicAdd(p.counters + EQ_PING + threadIdx.x, (unsigned long long)s_cnt[threadIdx.x]);
}

/* a node made pending; counted when it was neither pending nor removed */
__device__ __forceinline__ void wk_pend(const WalkEvParams &wp, uint64_t j)
{
    const uint32_t old = atomicOr(wp.mark + j, WK_PENDING);
    if (!(old & (WK_PENDING | WK_REMOVED)))
        atomicAdd(wp.mcount + WM_PENDING, 1ull);
}

__global__ void __launch_bounds__(256) regk_walk_mark_kernel(const WalkEvParams wp)
{
    const uint64_t e = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (e >= wp.n_ev)
        return;
    const uint64_t j = wp.node[e];
    if (j == ~0ull)
        return;
    if (wp.e.type[e] != 2) {
        wk_pend(wp, j);
        return;
    }
    const uint32_t old = atomicOr(wp.mark + j, WK_REMOVED);
    if (!(old & WK_REMOVED)) {
        atomicAdd(wp.mcount + WM_REMOVED, 1ull);
        if (old & WK_PENDING)
            atomicAdd(wp.mcount + WM_PENDING, ~0ull);           /* it leaves the pending set */
    }
    if (wp.parent[e] != ~0ull)
        wk_pend(wp, wp.parent[e]);
}

/* ---- apply: a refresh-level read's getData replies onto frontier node i's snapshot node fnode[i] ---- */
struct WalkApplyParams {
    uint64_t f;
    const unsigned long long *fnode;
    const int32_t *err, *ver;
    const long long *own;
    const unsigned long long *data_pos;
    const uint32_t *dlen;
    uint32_t *mark;
    int32_t *snap_ver;
    long long *snap_own;
    unsigned long long *rpos;                   /* [m] where a replaced node's data lies in the reply stream */
    uint32_t *rlen;
};

__global__ void __launch_bounds__(256) regk_walk_apply_kernel(const WalkApplyParams p)
{
    const uint64_t i = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= p.f)
        return;
    const uint64_t j = p.fnode[i];
    const int32_t e = p.err[i];
    if (e == 0) {
        p.snap_ver[j] = p.ver[i];
        p.snap_own[j] = p.own[i];
        p.rpos[j] = p.data_pos[i];
        p.rlen[j] = p.dlen[i];
        p.mark[j] |= WK_REPLACED;
    } else if (e == -101) {
        p.mark[j] |= WK_REMOVED;
    }
}

/* ---- keep: the nodes not marked removed, in order, with their sources, version, owner and mark ---- */
struct WalkKeepParams {
    uint64_t m;
    const uint32_t *mark;
    const unsigned long long *path_off, *json_off;
    const int32_t *ver;
    const long long *own;
    const unsigned long long *rpos;             /* read where mark & WK_REPLACED */
    const uint32_t *rlen;
    uint32_t *tile_total;
    unsigned long long *super_total;
    unsigned long long *counters;               /* [2]: kept, kept pending */
    unsigned long long *psrc, *dsrc;            /* [kept] */
    uint32_t *plen, *dlen;
    uint8_t *dsel;                              /* 1: the data comes from the reply stream */
    uint32_t *nmark;
    int32_t *nver;
    long long *nown;
};

__global__ void __launch_bounds__(RP_TILE) regk_walk_keep_count_kernel(const WalkKeepParams p)
{
    __shared__ uint32_t s_cnt[2];
    if (threadIdx.x < 2)
        s_cnt[threadIdx.x] = 0;
    __syncthreads();
    const uint64_t j = (uint64_t)blockIdx.x * RP_TILE + threadIdx.x;
    const uint32_t mk = j < p.m ? p.mark[j] : WK_REMOVED;
    const bool keep = !(mk & WK_REMOVED);
    const uint32_t cnt = (uint32_t)__popc(__ballot_sync(0xFFFFFFFFu, keep));
    if ((threadIdx.x & 31u) == 0)
        add_tile_total(p.tile_total, p.super_total, blockIdx.x, cnt);
    if (keep)
        atomicAdd(&s_cnt[0], 1u);
    if (keep && (mk & WK_PENDING))
        atomicAdd(&s_cnt[1], 1u);
    __syncthreads();
    if (threadIdx.x < 2 && s_cnt[threadIdx.x])
        atomicAdd(p.counters + threadIdx.x, (unsigned long long)s_cnt[threadIdx.x]);
}

__global__ void __launch_bounds__(RP_TILE) regk_walk_keep_kernel(const WalkKeepParams p)
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
    if (keep) {
        const uint64_t k = s_base + r;
        const bool rep = mk & WK_REPLACED;
        p.psrc[k] = p.path_off[j];
        p.plen[k] = (uint32_t)(p.path_off[j + 1] - p.path_off[j]);
        p.dsrc[k] = rep ? p.rpos[j] : p.json_off[j];
        p.dlen[k] = rep ? p.rlen[j] : (uint32_t)(p.json_off[j + 1] - p.json_off[j]);
        p.dsel[k] = rep ? 1u : 0u;
        p.nmark[k] = mk & WK_PENDING;
        p.nver[k] = p.ver[j];
        p.nown[k] = p.own[j];
    }
}

/* ---- rebuild: item k's len[k] bytes from src[sel[k]] at src_off[k], packed; output-stationary 16-byte blocks ---- */
struct WalkRebuildParams {
    uint64_t n;
    const uint8_t *src0, *src1;
    const unsigned long long *src_off;
    const uint8_t *sel;                         /* NULL: every item from src0 */
    const uint32_t *len;
    const unsigned long long *tile_total;       /* regk_mkdirp_len_kernel's totals of len */
    const unsigned long long *super_total;
    uint8_t *out;
    unsigned long long *out_off;                /* [n + 1] */
};

__global__ void __launch_bounds__(MK_TILE) regk_walk_rebuild_kernel(const WalkRebuildParams p)
{
    __shared__ unsigned long long s_warp[MK_TILE / 32];
    __shared__ unsigned long long s_off[MK_TILE + 1];           /* tile-relative byte offsets */
    __shared__ unsigned long long s_src[MK_TILE];               /* where each item's bytes start in its source */
    __shared__ uint8_t s_sel[MK_TILE];
    __shared__ unsigned long long s_base;
    const uint32_t tile = blockIdx.x, lane = threadIdx.x & 31u;
    if (threadIdx.x < 32) {
        const uint32_t nsuper = tile / SUPER;
        unsigned long long acc = 0;
        for (uint32_t i = lane; i < nsuper; i += 32)
            acc += p.super_total[i];
        for (uint32_t i = nsuper * SUPER + lane; i < tile; i += 32)
            acc += p.tile_total[i];
        #pragma unroll
        for (int d = 16; d > 0; d >>= 1)
            acc += __shfl_xor_sync(0xFFFFFFFFu, acc, d);
        if (lane == 0)
            s_base = acc;
    }
    const uint64_t k0 = (uint64_t)tile * MK_TILE, k = k0 + threadIdx.x;
    const uint32_t nd = (uint32_t)min((uint64_t)MK_TILE, p.n - k0);
    const unsigned long long len = threadIdx.x < nd ? p.len[k] : 0ull;
    if (threadIdx.x < nd) {
        s_src[threadIdx.x] = p.src_off[k];
        s_sel[threadIdx.x] = p.sel ? p.sel[k] : (uint8_t)0;
    }
    unsigned long long total;
    const unsigned long long excl = block_scan<unsigned long long>(s_warp, len, &total);   /* barriers: s_base, s_src */
    const unsigned long long base = s_base;
    if (threadIdx.x < nd) {
        s_off[threadIdx.x] = excl;
        p.out_off[k] = base + excl;
    }
    if (threadIdx.x == 0)
        s_off[nd] = total;
    if (k0 + nd == p.n && threadIdx.x == 0)
        p.out_off[p.n] = base + total;
    __syncthreads();
    const unsigned long long a0 = base & ~15ull;
    const uint32_t lead = (uint32_t)(base - a0);
    const unsigned long long nblk = (lead + total + 15ull) >> 4;
    for (unsigned long long b = threadIdx.x; b < nblk; b += MK_TILE) {
        const long long bs = (long long)(16ull * b) - (long long)lead;   /* tile-relative byte of the block's lane 0 */
        const unsigned long long pos0 = bs < 0 ? 0ull : (unsigned long long)bs;
        const unsigned long long end = min((unsigned long long)(bs + 16), total);
        uint32_t lo = 0, hi = nd - 1u;                          /* the item pos0 lies in: last s_off[d] <= pos0 */
        while (lo < hi) {
            const uint32_t mid = (lo + hi + 1u) >> 1;
            if (s_off[mid] <= pos0)
                lo = mid;
            else
                hi = mid - 1u;
        }
        uint32_t d = lo;
        uint32_t acc[4] = {0u, 0u, 0u, 0u};
        for (unsigned long long q = pos0; q < end; q++) {
            while (q >= s_off[d + 1])
                d++;
            const uint8_t *src = s_sel[d] ? p.src1 : p.src0;
            const uint32_t byte = src[s_src[d] + (q - s_off[d])];
            const uint32_t lanebyte = (uint32_t)(q - (unsigned long long)bs);
            acc[lanebyte >> 2] |= byte << (8u * (lanebyte & 3u));
        }
        uint8_t *gp = p.out + a0 + 16ull * b;
        if (bs >= 0 && (unsigned long long)bs + 16ull <= total) {
            stg_v4(gp, make_uint4(acc[0], acc[1], acc[2], acc[3]));
        } else {                                                /* the tile's ragged first / last block: its own bytes only */
            for (unsigned long long q = pos0; q < end; q++) {
                const uint32_t lanebyte = (uint32_t)(q - (unsigned long long)bs);
                gp[lanebyte] = (uint8_t)(acc[lanebyte >> 2] >> (8u * (lanebyte & 3u)));
            }
        }
    }
}

/* ---- filter: listing entry e stays iff its path is not a snapshot node (with skip_removed: not an unmarked one) ---- */
struct WalkFilterParams {
    uint64_t n;
    const uint8_t *lbytes;                      /* the listing's packed paths, readable below ltotal */
    const unsigned long long *loff;
    uint64_t ltotal;
    const uint8_t *spath;
    const unsigned long long *soff;
    const uint32_t *table;
    uint32_t mask;
    const uint32_t *mark;
    uint32_t skip_removed;                      /* 1: a node marked removed does not count */
    uint32_t *tile_total;
    unsigned long long *super_total;
    uint8_t *keep;                              /* [n] */
    unsigned long long *rec, *count;            /* [kept] entry, and the kept count */
    uint32_t *len;
};

__global__ void __launch_bounds__(RP_TILE) regk_walk_filter_count_kernel(const WalkFilterParams p)
{
    const uint64_t e = (uint64_t)blockIdx.x * RP_TILE + threadIdx.x;
    bool keep = false;
    if (e < p.n) {
        const unsigned long long o = p.loff[e];
        const uint64_t j = wk_find(p.table, p.mask, p.spath, p.soff, reinterpret_cast<const uint32_t *>(p.lbytes), o,
                                   p.ltotal, (uint32_t)(p.loff[e + 1] - o));
        keep = j == ~0ull || (p.skip_removed && (p.mark[j] & WK_REMOVED));
        p.keep[e] = keep ? 1u : 0u;
    }
    const uint32_t cnt = (uint32_t)__popc(__ballot_sync(0xFFFFFFFFu, keep));
    if ((threadIdx.x & 31u) == 0)
        add_tile_total(p.tile_total, p.super_total, blockIdx.x, cnt);
}

__global__ void __launch_bounds__(RP_TILE) regk_walk_filter_kernel(const WalkFilterParams p)
{
    __shared__ uint32_t s_warp[WARPS];
    __shared__ unsigned long long s_base;
    if (threadIdx.x < 32) {
        const unsigned long long base = tile_base_from_totals(p.tile_total, p.super_total, blockIdx.x);
        if (threadIdx.x == 0)
            s_base = base;
    }
    const uint64_t e = (uint64_t)blockIdx.x * RP_TILE + threadIdx.x;
    const bool keep = e < p.n && p.keep[e];
    uint32_t tot;
    const uint32_t r = block_scan<uint32_t>(s_warp, keep ? 1u : 0u, &tot);     /* its barriers publish s_base */
    if (keep) {
        const uint64_t k = s_base + r;
        p.rec[k] = e;
        p.len[k] = (uint32_t)(p.loff[e + 1] - p.loff[e]);
    }
    if (e + 1 == p.n)
        *p.count = s_base + tot;
}

}  /* namespace regk */
#endif /* REGK_WALK_WATCH_CUH */
