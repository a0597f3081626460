/*
 * regk_setwatches.cuh — keep the watched heartbeat's watches across a reconnect: frame one or more SetWatches requests
 * (op 101) for the watches the session holds, re-pend what they cannot cover (regk_setwatches_requests), and let
 * regk_read_events accept the SetWatches replies (xid -8) once such a framing was made.
 *
 * PARITY UNPINNED: the layout is restated from zookeeper.jute (RequestHeader, SetWatches) and tested against an
 * independent restatement, not against a server.  A frame, big endian:
 *   int len | int xid = -8 | int type = 101 | long relativeZxid | int nD | nD x (int P | path) | int nE | ... | int nC | ...
 * so a frame is 32 bytes of header and count words plus its entries.  Entry j of S = D ++ E ++ C is 4 + P bytes; s_j is
 * the exclusive prefix of those sizes; with B = max_frame - 32 - Lmax (Lmax = 4 + the batch's longest path) entry j
 * goes into frame floor(s_j / B).  Frame f starts at 32 f + s_first(f) and entry j at sw_entry_pos(s_j, B, list).
 * The reply is a bare ReplyHeader: len == 16, xid -8, err 0.
 *
 * ev_sw_head() / ev_sw_mask16() are ev_head() / ev_mask16() with a SetWatches reply as a fourth kind of frame; host +
 * device code (the CPU tests run them).  regk_read_events uses them, and regk_events_sw_cand_kernel, only after a
 * successful regk_setwatches_requests for the batch, so without one every frame is judged exactly as before.
 *
 * framing   lmax (the longest path, once per batch generation), classify (one thread per record and per directory:
 *           its list, or its re-pend mark, and per-tile counts and bytes of each list), place (the tile look-back of
 *           those totals: each entry's index j, s_j, path and length), write (the entries' bytes, output-stationary:
 *           every 16-byte block of a tile's span assembled in registers) and head (one thread per frame: its header,
 *           its three count words and its offset).
 */
#ifndef REGK_SETWATCHES_CUH
#define REGK_SETWATCHES_CUH

#include "regk_events.cuh"

namespace regk {

/* ev_sw_head results beyond ev_head's */
enum : uint32_t {
    EV_SW_BODY = EV_PING_BODY + 1,      /* a SetWatches reply with len != 16 */
    EV_SW_ERR,                          /* a SetWatches reply with err != 0 */
};

constexpr int32_t SW_XID = -8;
constexpr int32_t SW_OP = 101;
constexpr uint64_t SW_OVERHEAD = 32;    /* header (len, xid, type, relativeZxid) and the three count words */
constexpr int32_t ZK_NONODE = -101;

/* watch kinds: what the session's last read of a record or directory armed */
enum : uint8_t { WK_NONE = 0, WK_DATA = 1, WK_EXIST = 2, WK_CHILD = 3 };
/* lists of a SetWatches framing */
enum : uint32_t { SW_LIST_D = 0, SW_LIST_E = 1, SW_LIST_C = 2 };

RG_HD uint32_t ev_sw_words(int32_t L, int32_t xid, int32_t err, int32_t type, int32_t P, int32_t xid_base, uint64_t n)
{
    if (xid == SW_XID)
        return L != 16 ? (uint32_t)EV_SW_BODY : err != 0 ? (uint32_t)EV_SW_ERR : (uint32_t)EV_OK;
    return ev_words(L, xid, err, type, P, xid_base, n);
}

RG_HD uint32_t ev_sw_head(const uint8_t *b, uint64_t avail, int32_t xid_base, uint64_t n, EvHead *h)
{
    const uint32_t c = ev_head(b, avail, xid_base, n, h);
    if (c == EV_TRUNC || c == EV_BAD_LEN || h->xid != SW_XID)
        return c;
    return h->len != 16 ? (uint32_t)EV_SW_BODY : h->err != 0 ? (uint32_t)EV_SW_ERR : (uint32_t)EV_OK;
}

RG_HD uint32_t ev_sw_mask16(const uint32_t *w, uint64_t avail, uint32_t first, int32_t xid_base, uint64_t n)
{
    const uint32_t room = avail > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)avail;
    uint32_t mask = 0;
#if defined(__CUDA_ARCH__)
    #pragma unroll
#endif
    for (uint32_t f = 0; f < 16u; f++) {
        const uint32_t q = f >> 2, sh = f & 3u;
        const int32_t L = (int32_t)st_be32(w[q], w[q + 1], sh);
        const int32_t xid = (int32_t)st_be32(w[q + 1], w[q + 2], sh);
        const int32_t err = (int32_t)st_be32(w[q + 4], w[q + 5], sh);
        const int32_t type = (int32_t)st_be32(w[q + 5], w[q + 6], sh);
        const int32_t P = (int32_t)st_be32(w[q + 7], w[q + 8], sh);
        const bool fits = f >= first && L >= 16 && (uint32_t)L + 4u + f <= room;
        if (fits && ev_sw_words(L, xid, err, type, P, xid_base, n) == EV_OK)
            mask |= 1u << f;
    }
    return mask;
}

/* where entry j (s_j = the sizes 4 + P of the entries before it; list = SW_LIST_*) lands in the framing's bytes */
RG_HD uint64_t sw_entry_pos(uint64_t s_j, uint64_t B, uint32_t list)
{
    return s_j + SW_OVERHEAD * (s_j / B) + 24u + (list != SW_LIST_D ? 4u : 0u) + (list == SW_LIST_C ? 4u : 0u);
}

/* the first byte of frame f, whose first entry has prefix s_first */
RG_HD uint64_t sw_frame_off(uint64_t f, uint64_t s_first)
{
    return SW_OVERHEAD * f + s_first;
}

}  /* namespace regk */

#if defined(__CUDACC__)

namespace regk {

/* ---- cand with SetWatches replies: regk_events_cand_kernel's test through ev_sw_mask16 ---- */
__global__ void __launch_bounds__(RP_TILE) regk_events_sw_cand_kernel(const EvParams ep)
{
    const RepParams &p = ep.r;
    __shared__ uint32_t s_warp[WARPS];
    const uint64_t nblk = (p.len + 15u) / 16u;
    const uint64_t b = (uint64_t)blockIdx.x * RP_TILE + threadIdx.x;
    uint32_t mask = 0;
    if (b < nblk && 16ull * b + 16u > ep.start) {
        const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
        const uint4 v0 = rp_block(p.s, p.len, b);
        const uint4 v1 = b + 1 < nblk ? rp_block(p.s, p.len, b + 1) : zero;
        const uint4 v2 = b + 2 < nblk ? rp_block(p.s, p.len, b + 2) : zero;
        const uint32_t w[12] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w, v2.x, v2.y, v2.z, v2.w};
        const uint64_t at = 16ull * b;
        mask = ev_sw_mask16(w, p.len - at, ep.start > at ? (uint32_t)(ep.start - at) : 0u, p.xid_base, p.n);
    }
    uint32_t total;
    const uint32_t rank = block_scan<uint32_t>(s_warp, (uint32_t)__popc(mask), &total);
    if (b < nblk)
        p.word[b] = mask | rank << 16;
    if (threadIdx.x == 0)
        add_tile_total(p.tile_total, p.super_total, blockIdx.x, total);
}

/* ---- the session's zxid high-water mark: the largest ReplyHeader.zxid of the chain's replies (every frame but
   notifications and pings) ---- */
__global__ void __launch_bounds__(256) regk_events_zxid_kernel(const RepParams p, long long *zmax)
{
    const uint64_t c = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    long long z = 0;
    if (c < p.C && p.marked[c]) {
        const uint8_t *fr = p.s + p.cand[c];
        const int32_t xid = (int32_t)be32_at(fr + 4);
        if (xid != -1 && xid != -2)
            z = st_be64_at(fr + 8);
    }
    #pragma unroll
    for (int d = 16; d > 0; d >>= 1)
        z = max(z, (long long)__shfl_xor_sync(0xFFFFFFFFu, z, d));
    if ((threadIdx.x & 31u) == 0 && z > 0)
        atomicMax(zmax, z);
}

/* ---- watch kinds from a watched read: item sub[k] (or k) gets the kind its reply's err arms ---- */
struct WatchKindParams {
    uint64_t m;
    const int32_t *err;                         /* [m] */
    const unsigned long long *sub;              /* [m] the subset's items, NULL: item k */
    uint8_t *kind;
    bool dirs;
};

__global__ void __launch_bounds__(256) regk_watch_kind_kernel(const WatchKindParams p)
{
    const uint64_t k = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (k >= p.m)
        return;
    const int32_t e = p.err[k];
    const uint8_t kd = p.dirs ? (e == 0 ? WK_CHILD : WK_NONE) : (e == 0 ? WK_DATA : e == ZK_NONODE ? WK_EXIST : WK_NONE);
    p.kind[p.sub ? p.sub[k] : k] = kd;
}

/* ---- in flight: the items of an unread watched subset framing count as NONE ---- */
__global__ void __launch_bounds__(256) regk_watch_forget_kernel(const unsigned long long *items, uint64_t m, uint8_t *kind)
{
    const uint64_t k = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (k < m)
        kind[items[k]] = WK_NONE;
}

/* ---- lmax: the longest path of the batch ---- */
__global__ void __launch_bounds__(256) regk_sw_lmax_kernel(const unsigned long long *path_off, uint64_t n, uint32_t *lmax)
{
    const uint64_t i = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    uint32_t L = i < n ? (uint32_t)(path_off[i + 1] - path_off[i]) : 0u;
    L = __reduce_max_sync(0xFFFFFFFFu, L);
    if ((threadIdx.x & 31u) == 0 && L)
        atomicMax(lmax, L);
}

/* tile totals of the framing: record tiles D count, E count, D bytes, E bytes; directory tiles C count, C bytes */
enum { SWT_DC = 0, SWT_EC, SWT_DB, SWT_EB, SWT_CC, SWT_CB, SWT_N };
enum { SWQ_REPEND_R = 0, SWQ_REPEND_D, SWQ_N };

struct SwParams {
    uint64_t n, d;
    uint32_t tiles_r;                           /* CTAs over the records; the directories' CTAs follow */
    const unsigned long long *path_off;
    const uint32_t *slot, *t_rec;               /* the record table: record i is first of its path iff t_rec[slot[i]] == i + 1 */
    const unsigned long long *dir_rec;
    const uint32_t *dir_len;
    const uint8_t *rec_kind, *dir_kind;
    uint32_t *rec_mark, *dir_mark;
    uint32_t rec_epoch, dir_epoch;
    unsigned long long *dirty;                  /* [2] pending records, directories */
    unsigned long long *counters;               /* [SWQ_N] */
    uint8_t *cls;                               /* [n + d] 1 + SW_LIST_* of a listed item, 0 otherwise */
    uint32_t *tt[SWT_N];
    unsigned long long *st[SWT_N];
    /* place, write, head */
    uint64_t nD, nE, m, bD, bE, total_s, B;
    long long zxid;
    unsigned long long *ent_src, *ent_s;        /* [m] where each entry's path starts in path_bytes, s_j */
    uint32_t *ent_len;
    const uint8_t *path_bytes;
    uint8_t *out;
    unsigned long long *frame_off;              /* [F + 1] */
    uint64_t F;
};

/* item t of CTA `blk`: a record (i) or a directory (k); its list (1 + SW_LIST_*, 0 = none) and entry size */
__device__ __forceinline__ bool sw_item(const SwParams &p, uint32_t blk, uint64_t *idx, bool *dir)
{
    *dir = blk >= p.tiles_r;
    *idx = (uint64_t)(*dir ? blk - p.tiles_r : blk) * RP_TILE + threadIdx.x;
    return *idx < (*dir ? p.d : p.n);
}

__global__ void __launch_bounds__(RP_TILE) regk_sw_classify_kernel(const SwParams p)
{
    uint64_t i;
    bool dir;
    const bool on = sw_item(p, blockIdx.x, &i, &dir);
    uint32_t list = 0, size = 0;
    bool repend = false;
    if (on && !dir) {
        const bool first = p.t_rec[p.slot[i]] == (uint32_t)i + 1u;
        const bool pend = (p.rec_mark[i] >> 3) == p.rec_epoch;
        if (first && !pend) {
            const uint8_t k = p.rec_kind[i];
            if (k == WK_DATA || k == WK_EXIST) {
                list = 1u + (k == WK_DATA ? SW_LIST_D : SW_LIST_E);
                size = 4u + (uint32_t)(p.path_off[i + 1] - p.path_off[i]);
            } else {
                repend = true;
                p.rec_mark[i] = p.rec_epoch << 3;
            }
        }
    } else if (on) {
        if (p.dir_mark[i] != p.dir_epoch) {
            if (p.dir_kind[i] == WK_CHILD) {
                list = 1u + SW_LIST_C;
                size = 4u + p.dir_len[i];
            } else {
                repend = true;
                p.dir_mark[i] = p.dir_epoch;
            }
        }
    }
    if (on)
        p.cls[dir ? p.n + i : i] = (uint8_t)list;
    const uint32_t nrep = __popc(__ballot_sync(0xFFFFFFFFu, repend));
    const uint32_t c0 = __popc(__ballot_sync(0xFFFFFFFFu, list == 1u + SW_LIST_D || list == 1u + SW_LIST_C));
    const uint32_t c1 = __popc(__ballot_sync(0xFFFFFFFFu, list == 1u + SW_LIST_E));
    const uint32_t b0 = __reduce_add_sync(0xFFFFFFFFu, list == 1u + SW_LIST_E ? 0u : size);
    const uint32_t b1 = __reduce_add_sync(0xFFFFFFFFu, list == 1u + SW_LIST_E ? size : 0u);
    if ((threadIdx.x & 31u) == 0) {
        const uint32_t t = dir ? blockIdx.x - p.tiles_r : blockIdx.x;
        if (dir) {
            add_tile_total(p.tt[SWT_CC], p.st[SWT_CC], t, c0);
            add_tile_total(p.tt[SWT_CB], p.st[SWT_CB], t, b0);
        } else {
            add_tile_total(p.tt[SWT_DC], p.st[SWT_DC], t, c0);
            add_tile_total(p.tt[SWT_EC], p.st[SWT_EC], t, c1);
            add_tile_total(p.tt[SWT_DB], p.st[SWT_DB], t, b0);
            add_tile_total(p.tt[SWT_EB], p.st[SWT_EB], t, b1);
        }
        if (nrep) {
            atomicAdd(p.dirty + (dir ? 1 : 0), (unsigned long long)nrep);
            atomicAdd(p.counters + (dir ? SWQ_REPEND_D : SWQ_REPEND_R), (unsigned long long)nrep);
        }
    }
}

/* ---- place: each listed item's entry index j and prefix s_j, from its CTA's look-back and an in-CTA scan ---- */
__global__ void __launch_bounds__(RP_TILE) regk_sw_place_kernel(const SwParams p)
{
    __shared__ unsigned long long s_warp[WARPS];
    __shared__ unsigned long long s_base[4];
    uint64_t i;
    bool dir;
    const bool on = sw_item(p, blockIdx.x, &i, &dir);
    const uint32_t t = dir ? blockIdx.x - p.tiles_r : blockIdx.x;
    if (threadIdx.x < 32) {
        /* the look-back: list counts and bytes of the CTAs before this one */
        const int a[4] = {dir ? SWT_CC : SWT_DC, dir ? SWT_CB : SWT_DB, SWT_EC, SWT_EB};
        for (int q = 0; q < (dir ? 2 : 4); q++) {
            const unsigned long long v = tile_base_from_totals(p.tt[a[q]], p.st[a[q]], t);
            if (threadIdx.x == 0)
                s_base[q] = v;
        }
    }
    const uint32_t list = on ? p.cls[dir ? p.n + i : i] : 0u;
    const uint64_t rec = on ? (dir ? p.dir_rec[i] : i) : 0;
    const uint32_t P = !list ? 0u : dir ? p.dir_len[i] : (uint32_t)(p.path_off[i + 1] - p.path_off[i]);
    /* one scan of count << 40 | bytes per list; a CTA's bytes stay below 2^40 */
    const bool e = list == 1u + SW_LIST_E;
    const unsigned long long v = list ? (1ull << 40) | (4ull + P) : 0ull;
    unsigned long long tot;
    const unsigned long long x0 = block_scan<unsigned long long>(s_warp, e ? 0ull : v, &tot);  /* barriers: s_base */
    __syncthreads();
    const unsigned long long x1 = dir ? 0ull : block_scan<unsigned long long>(s_warp, e ? v : 0ull, &tot);
    if (!list)
        return;
    const unsigned long long x = e ? x1 : x0;
    const uint64_t rank = x >> 40, rb = x & ((1ull << 40) - 1);
    uint64_t j, s;
    if (dir) {
        j = p.nD + p.nE + s_base[0] + rank;
        s = p.bD + p.bE + s_base[1] + rb;
    } else if (!e) {
        j = s_base[0] + rank;
        s = s_base[1] + rb;
    } else {
        j = p.nD + s_base[2] + rank;
        s = p.bD + s_base[3] + rb;
    }
    p.ent_src[j] = p.path_off[rec];
    p.ent_len[j] = P;
    p.ent_s[j] = s;
}

__device__ __forceinline__ uint32_t sw_list_of(const SwParams &p, uint64_t j)
{
    return j < p.nD ? SW_LIST_D : j < p.nD + p.nE ? SW_LIST_E : SW_LIST_C;
}

/* ---- write: the entries (int P | path), output-stationary over each CTA's span; bytes between entries (count words
   and headers) are left to the head kernel, which runs after ---- */
__global__ void __launch_bounds__(RP_TILE) regk_sw_write_kernel(const SwParams p)
{
    __shared__ unsigned long long s_pos[RP_TILE + 1];       /* span-relative entry starts; [nd] = the span's end */
    __shared__ unsigned long long s_src[RP_TILE];
    __shared__ uint32_t s_len[RP_TILE];
    const uint64_t k0 = (uint64_t)blockIdx.x * RP_TILE, k = k0 + threadIdx.x;
    const uint32_t nd = (uint32_t)min((uint64_t)RP_TILE, p.m - k0);
    const uint64_t base = sw_entry_pos(p.ent_s[k0], p.B, sw_list_of(p, k0));
    if (threadIdx.x < nd) {
        const uint32_t P = p.ent_len[k];
        const uint64_t pos = sw_entry_pos(p.ent_s[k], p.B, sw_list_of(p, k));
        s_pos[threadIdx.x] = pos - base;
        s_src[threadIdx.x] = p.ent_src[k];
        s_len[threadIdx.x] = P;
        if (threadIdx.x == nd - 1)
            s_pos[nd] = pos + 4u + P - base;
    }
    __syncthreads();
    const unsigned long long total = s_pos[nd];
    const unsigned long long a0 = base & ~15ull;
    const uint32_t lead = (uint32_t)(base - a0);
    const unsigned long long nblk = (lead + total + 15ull) >> 4;
    for (unsigned long long b = threadIdx.x; b < nblk; b += RP_TILE) {
        const long long bs = (long long)(16ull * b) - (long long)lead;     /* span-relative byte of the block's lane 0 */
        const unsigned long long pos0 = bs < 0 ? 0ull : (unsigned long long)bs;
        const unsigned long long end = min((unsigned long long)(bs + 16), total);
        uint32_t lo = 0, hi = nd - 1u;                                  /* the entry pos0 lies in or after */
        while (lo < hi) {
            const uint32_t mid = (lo + hi + 1u) >> 1;
            if (s_pos[mid] <= pos0)
                lo = mid;
            else
                hi = mid - 1u;
        }
        uint32_t d = lo;
        unsigned long long acc0 = 0, acc1 = 0;                          /* the block's bytes 0 .. 7 and 8 .. 15 */
        for (unsigned long long q = pos0; q < end; q++) {
            while (q >= s_pos[d + 1])
                d++;
            const unsigned long long r = q - s_pos[d];
            uint32_t byte = 0;
            if (r < 4u)
                byte = (s_len[d] >> (8u * (3u - (uint32_t)r))) & 0xFFu;
            else if (r < 4ull + s_len[d])
                byte = p.path_bytes[s_src[d] + (r - 4u)];
            const uint32_t lanebyte = (uint32_t)(q - (unsigned long long)bs);
            if (lanebyte < 8u)
                acc0 |= (unsigned long long)byte << (8u * lanebyte);
            else
                acc1 |= (unsigned long long)byte << (8u * (lanebyte - 8u));
        }
        uint8_t *gp = p.out + a0 + 16ull * b;
        if (bs >= 0 && (unsigned long long)bs + 16ull <= total) {
            stg_v4(gp, make_uint4((uint32_t)acc0, (uint32_t)(acc0 >> 32), (uint32_t)acc1, (uint32_t)(acc1 >> 32)));
        } else {                                                        /* the span's ragged first / last block */
            for (unsigned long long q = pos0; q < end; q++) {
                const uint32_t lanebyte = (uint32_t)(q - (unsigned long long)bs);
                gp[lanebyte] = (uint8_t)(lanebyte < 8u ? acc0 >> (8u * lanebyte) : acc1 >> (8u * (lanebyte - 8u)));
            }
        }
    }
}

__device__ __forceinline__ void sw_put32(uint8_t *b, uint32_t v)
{
    b[0] = (uint8_t)(v >> 24);
    b[1] = (uint8_t)(v >> 16);
    b[2] = (uint8_t)(v >> 8);
    b[3] = (uint8_t)v;
}

/* the first entry j with s_j >= v (m when none) */
__device__ __forceinline__ uint64_t sw_lower(const SwParams &p, uint64_t v)
{
    uint64_t lo = 0, hi = p.m;
    while (lo < hi) {
        const uint64_t mid = (lo + hi) >> 1;
        if (p.ent_s[mid] < v)
            lo = mid + 1;
        else
            hi = mid;
    }
    return lo;
}

/* ---- head: frame f's header and count words, and its offset ---- */
__global__ void __launch_bounds__(256) regk_sw_head_kernel(const SwParams p)
{
    const uint64_t f = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (f >= p.F)
        return;
    const uint64_t j0 = sw_lower(p, f * p.B), j1 = f + 1 == p.F ? p.m : sw_lower(p, (f + 1) * p.B);
    auto s_at = [&](uint64_t j) { return j < p.m ? (uint64_t)p.ent_s[j] : p.total_s; };
    auto clampj = [&](uint64_t j) { return j < j0 ? j0 : j > j1 ? j1 : j; };
    const uint64_t dEnd = clampj(p.nD), eEnd = clampj(p.nD + p.nE);
    const uint64_t s0 = s_at(j0), sd = s_at(dEnd), se = s_at(eEnd), s1 = s_at(j1);
    const uint64_t off = sw_frame_off(f, s0);
    uint8_t *fr = p.out + off;
    sw_put32(fr, (uint32_t)(SW_OVERHEAD + (s1 - s0) - 4u));
    sw_put32(fr + 4, (uint32_t)SW_XID);
    sw_put32(fr + 8, (uint32_t)SW_OP);
    sw_put32(fr + 12, (uint32_t)((unsigned long long)p.zxid >> 32));
    sw_put32(fr + 16, (uint32_t)p.zxid);
    sw_put32(fr + 20, (uint32_t)(dEnd - j0));
    sw_put32(fr + 24 + (sd - s0), (uint32_t)(eEnd - dEnd));
    sw_put32(fr + 28 + (se - s0), (uint32_t)(j1 - eEnd));
    p.frame_off[f] = off;
    if (f + 1 == p.F)
        p.frame_off[p.F] = SW_OVERHEAD * p.F + p.total_s;
}

}  /* namespace regk */
#endif /* __CUDACC__ */
#endif /* REGK_SETWATCHES_CUH */
