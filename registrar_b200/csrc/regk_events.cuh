/*
 * regk_events.cuh — the watched heartbeat: read ZooKeeper's watch notifications on the GPU, map each one to the record
 * or service directory it is about, and keep the records and directories that fired as a pending set the re-arming
 * requests are framed from (regk_read_events, regk_events_requests).
 *
 * PARITY UNPINNED: the layout is restated from zookeeper.jute (ReplyHeader, WatcherEvent) and tested against an
 * independent restatement, not against a server.  A notification frame, big endian:
 *   int len | int xid = -1 | long zxid | int err = 0 | WatcherEvent{int type; int state; ustring path}
 * so len == 28 + P, with type at 20, state at 24, the path length P at 28 and the path at 32 from the frame's first byte.
 * A ping is xid -2 with len == 16.  A frame whose xid lies in the caller's reply range is a reply to an outstanding
 * request: it is skipped by its length whatever its body.
 *
 * ev_head() is the full test of one position and ev_mask16() the same test for the 16 start phases of one 16-byte block
 * from words held in registers.  Both are host + device code (the CPU tests run them).  Every check is in the
 * plausibility test, so a chain frame needs no second check: the chain stops at the first position that fails it,
 * and the host names the reason there (or reports a partial trailing frame).
 *
 * reading   cand (ev_mask16() over every block at or after start), then regk_replies.cuh's compact, succ, jump and mark
 *           kernels and its stop kernel; count (the chain's notifications per CTA) and events (one thread per chain
 *           frame: a notification's fields, its path looked up in the record table and the directory table - compared
 *           byte for byte, a hash only picks a slot - and its subject marked in the per-generation arrays).
 * tables    built once per batch generation: the records by regk_replies_insert_kernel (the first record with a path
 *           keeps its slot, regk_reconcile_desired_kernel's protocol), the directories by dir_insert.
 * pending   a record is pending iff its mark's epoch (bits 3 and up) is the current one, a directory iff its mark is;
 *           regk_events_requests compacts the pending set in ascending order and starts the next epoch, so taking the
 *           set never clears n-sized state.
 */
#ifndef REGK_EVENTS_CUH
#define REGK_EVENTS_CUH

#include "regk_stats.cuh"

namespace regk {

/* ev_head results */
enum : uint32_t {
    EV_OK = 0,
    EV_TRUNC,           /* the stream ends inside the frame (or before its length word) */
    EV_BAD_LEN,         /* len < 16: no room for a ReplyHeader */
    EV_NEG_XID,         /* a negative xid other than -1 / -2, outside the reply range */
    EV_XID_RANGE,       /* a non-negative xid outside the reply range */
    EV_NOTE_LEN,        /* a notification whose length is not 28 + P */
    EV_NEG_PATH,        /* a notification with P < 0 */
    EV_NOTE_ERR,        /* a notification with err != 0 */
    EV_TYPE,            /* a notification whose type is outside -1 .. 7 */
    EV_PING_BODY,       /* a ping with len != 16 */
};

constexpr int32_t EV_NOTE_HEAD = 28;            /* the length word of a notification with an empty path */

struct EvHead {
    uint32_t kind;      /* RK_* */
    int32_t len, xid, err, type, plen;
};

/* the verdict on a position whose frame fits the stream, from its words (type and P matter only for xid -1) */
RG_HD uint32_t ev_words(int32_t L, int32_t xid, int32_t err, int32_t type, int32_t P, int32_t xid_base, uint64_t n)
{
    if (xid == -2)
        return L == 16 ? EV_OK : EV_PING_BODY;
    if (xid == -1) {
        if (L < EV_NOTE_HEAD)
            return EV_NOTE_LEN;
        if (P < 0)
            return EV_NEG_PATH;
        if (P != L - EV_NOTE_HEAD)
            return EV_NOTE_LEN;
        if (err != 0)
            return EV_NOTE_ERR;
        return type < -1 || type > 7 ? EV_TYPE : EV_OK;
    }
    if ((uint64_t)((uint32_t)xid - (uint32_t)xid_base) < n)
        return EV_OK;
    return xid < 0 ? EV_NEG_XID : EV_XID_RANGE;
}

/* The frame starting at b, with `avail` stream bytes from b on (reads at most 32 of them, never past avail and never
   past the frame): EV_OK when it is a notification, a ping or a reply in [xid_base, xid_base + n). */
RG_HD uint32_t ev_head(const uint8_t *b, uint64_t avail, int32_t xid_base, uint64_t n, EvHead *h)
{
    h->kind = RK_REPLY;
    h->len = h->xid = h->err = h->type = h->plen = 0;
    if (avail < 4)
        return EV_TRUNC;
    const int32_t L = (int32_t)be32_at(b);
    h->len = L;
    if (L < 16)
        return EV_BAD_LEN;
    if ((uint64_t)L + 4u > avail)
        return EV_TRUNC;
    h->xid = (int32_t)be32_at(b + 4);
    h->err = (int32_t)be32_at(b + 16);
    if (h->xid == -1 || h->xid == -2)
        h->kind = h->xid == -1 ? RK_NOTIFY : RK_PING;
    if (h->xid == -1 && L >= EV_NOTE_HEAD) {
        h->type = (int32_t)be32_at(b + 20);
        h->plen = (int32_t)be32_at(b + 28);
    }
    return ev_words(L, h->xid, h->err, h->type, h->plen, xid_base, n);
}

/* ev_head() == EV_OK for the 16 positions of one 16-byte block, as a bit mask.  w[0 .. 11] = the block and the 32
   bytes after it as little-endian words (bytes at or past the stream's end read as anything); avail = stream bytes
   from the block's first byte on; positions below `first` are left out. */
RG_HD uint32_t ev_mask16(const uint32_t *w, uint64_t avail, uint32_t first, int32_t xid_base, uint64_t n)
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
        if (fits && ev_words(L, xid, err, type, P, xid_base, n) == EV_OK)
            mask |= 1u << f;
    }
    return mask;
}

}  /* namespace regk */

#if defined(__CUDACC__)

namespace regk {

/* counters[]: regk_replies.cuh's (RQ_STOP is the stop kernel's), then these */
enum { EQ_NEV = RQ_NCOUNTERS, EQ_PING, EQ_REPLY, EQ_UNMATCHED, EQ_OTHER, EQ_NCOUNTERS };
enum : uint8_t { EV_SUBJ_NONE = 0, EV_SUBJ_RECORD = 1, EV_SUBJ_DIR = 2 };

struct EvParams {
    RepParams r;                                /* the frame chain; r.xid_base / r.n = the reply range */
    uint64_t start;
    /* the batch's paths, the record table (record + 1) and the directory table (directory + 1) */
    const uint8_t *d_path;
    const unsigned long long *d_path_off;
    const uint32_t *t_rec;
    uint32_t mask_r;
    const uint32_t *t_dir;
    uint32_t mask_d;
    const unsigned long long *dir_rec;
    const uint32_t *dir_len;
    /* per-generation marks and the pending counts (dirty[0] records, dirty[1] directories) */
    uint32_t *rec_mark;                         /* epoch << 3 | created 1 | deleted 2 | data 4 */
    uint32_t *dir_mark;                         /* epoch */
    uint32_t rec_epoch, dir_epoch;
    unsigned long long *dirty;
    /* the notification count pass's totals, and the events in stream order */
    uint32_t *tile_total;
    unsigned long long *super_total;
    unsigned long long *pos, *subject;
    int32_t *type, *state;
    long long *zxid;
    uint8_t *kind;
};

/* ---- cand: the plausible positions at or after start, 16 per thread, tested from registers ---- */
__global__ void __launch_bounds__(RP_TILE) regk_events_cand_kernel(const EvParams ep)
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
        mask = ev_mask16(w, p.len - at, ep.start > at ? (uint32_t)(ep.start - at) : 0u, p.xid_base, p.n);
    }
    uint32_t total;
    const uint32_t rank = block_scan<uint32_t>(s_warp, (uint32_t)__popc(mask), &total);
    if (b < nblk)
        p.word[b] = mask | rank << 16;
    if (threadIdx.x == 0)
        add_tile_total(p.tile_total, p.super_total, blockIdx.x, total);
}

__device__ __forceinline__ bool ev_is_note(const RepParams &p, uint64_t c)
{
    return c < p.C && p.marked[c] && (int32_t)be32_at(p.s + p.cand[c] + 4) == -1;
}

/* ---- count: the chain's notifications per CTA ---- */
__global__ void __launch_bounds__(RP_TILE) regk_events_count_kernel(const EvParams ep)
{
    const uint64_t c = (uint64_t)blockIdx.x * RP_TILE + threadIdx.x;
    const uint32_t cnt = (uint32_t)__popc(__ballot_sync(0xFFFFFFFFu, ev_is_note(ep.r, c)));
    if ((threadIdx.x & 31u) == 0)
        add_tile_total(ep.tile_total, ep.super_total, blockIdx.x, cnt);
}

/* the entry of `table` whose key is the n bytes at o of the stream V (readable below lim), or ~0 */
__device__ __forceinline__ uint64_t ev_find(const EvParams &ep, const uint32_t *table, uint32_t mask, bool dirs,
    const uint32_t *V, uint64_t o, uint64_t lim, uint32_t n)
{
    const uint32_t *W = reinterpret_cast<const uint32_t *>(ep.d_path);
    uint32_t slot = string_hash32_clamped(V, o, n, lim) & mask;
    for (;;) {
        const uint32_t cur = table[slot];
        if (cur == 0u)
            return ~0ull;
        const uint64_t k = cur - 1u;
        const uint64_t r = dirs ? ep.dir_rec[k] : k;
        const unsigned long long o0 = ep.d_path_off[r];
        const uint32_t L = dirs ? ep.dir_len[k] : (uint32_t)(ep.d_path_off[r + 1] - o0);
        if (L == n && string_equal2(W, o0, ~0ull, V, o, lim, n))
            return k;
        slot = (slot + 1u) & mask;
    }
}

/* ---- events: every chain notification's fields, its subject, and the mark; pings and replies counted ---- */
__global__ void __launch_bounds__(RP_TILE) regk_events_kernel(const EvParams ep)
{
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
        uint64_t subj = ~0ull;
        uint8_t kind = EV_SUBJ_NONE;
        if (type >= 1 && type <= 3) {
            subj = ev_find(ep, ep.t_rec, ep.mask_r, false, V, pos + 32u, p.len, P);
            if (subj != ~0ull) {
                kind = EV_SUBJ_RECORD;
                const uint32_t bit = 1u << (type - 1);
                uint32_t old = ep.rec_mark[subj];
                for (;;) {
                    const bool cur = (old >> 3) == ep.rec_epoch;
                    const uint32_t nw = cur ? old | bit : ep.rec_epoch << 3 | bit;
                    if (nw == old)
                        break;
                    const uint32_t prev = atomicCAS(ep.rec_mark + subj, old, nw);
                    if (prev == old) {
                        if (!cur)
                            atomicAdd(ep.dirty, 1ull);
                        break;
                    }
                    old = prev;
                }
            }
        }
        if (kind == EV_SUBJ_NONE && (type == 2 || type == 4)) {
            subj = ev_find(ep, ep.t_dir, ep.mask_d, true, V, pos + 32u, p.len, P);
            if (subj != ~0ull) {
                kind = EV_SUBJ_DIR;
                if (atomicExch(ep.dir_mark + subj, ep.dir_epoch) != ep.dir_epoch)
                    atomicAdd(ep.dirty + 1, 1ull);
            }
        }
        if (kind == EV_SUBJ_NONE)
            atomicAdd(&s_cnt[2], 1u);
        if (type == -1 || type >= 5)
            atomicAdd(&s_cnt[3], 1u);
        ep.pos[e] = pos;
        ep.type[e] = type;
        ep.state[e] = (int32_t)be32_at(fr + 24);
        ep.zxid[e] = st_be64_at(fr + 8);
        ep.kind[e] = kind;
        ep.subject[e] = subj;
    }
    if (c + 1 == p.C)
        p.counters[EQ_NEV] = s_base + tot;
    __syncthreads();
    if (threadIdx.x < 4 && s_cnt[threadIdx.x])
        atomicAdd(p.counters + EQ_PING + threadIdx.x, (unsigned long long)s_cnt[threadIdx.x]);
}

/* ---- the directory table: directory k + 1 under the hash of its path (the directories are distinct) ---- */
struct EvDirParams {
    const uint8_t *d_path;
    const unsigned long long *d_path_off;
    const unsigned long long *dir_rec;
    const uint32_t *dir_len;
    uint64_t d;
    uint32_t *table;
    uint32_t mask;
};

__global__ void __launch_bounds__(256) regk_events_dir_insert_kernel(const EvDirParams p)
{
    const uint64_t k = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (k >= p.d)
        return;
    const uint32_t *W = reinterpret_cast<const uint32_t *>(p.d_path);
    uint32_t slot = string_hash32(W, p.d_path_off[p.dir_rec[k]], p.dir_len[k]) & p.mask;
    while (atomicCAS(p.table + slot, 0u, (uint32_t)k + 1u) != 0u)
        slot = (slot + 1u) & p.mask;
}

/* ---- pending: the items whose mark >> shift is `epoch`, ascending; rec[k] / len[k] = the record and path length of
   item k (a directory's first record and length, or the record itself) ---- */
struct EvPendParams {
    uint64_t n;
    const uint32_t *mark;
    uint32_t shift, epoch;
    const unsigned long long *path_off;
    const unsigned long long *dir_rec;          /* NULL: the items are records */
    const uint32_t *dir_len;
    uint32_t *tile_total;
    unsigned long long *super_total;
    unsigned long long *item, *rec;
    uint32_t *len;
    unsigned long long *count;
};

__device__ __forceinline__ bool ev_pending(const EvPendParams &p, uint64_t i)
{
    return i < p.n && (p.mark[i] >> p.shift) == p.epoch;
}

__global__ void __launch_bounds__(RP_TILE) regk_events_pending_count_kernel(const EvPendParams p)
{
    const uint64_t i = (uint64_t)blockIdx.x * RP_TILE + threadIdx.x;
    const uint32_t cnt = (uint32_t)__popc(__ballot_sync(0xFFFFFFFFu, ev_pending(p, i)));
    if ((threadIdx.x & 31u) == 0)
        add_tile_total(p.tile_total, p.super_total, blockIdx.x, cnt);
}

__global__ void __launch_bounds__(RP_TILE) regk_events_pending_kernel(const EvPendParams p)
{
    __shared__ uint32_t s_warp[WARPS];
    __shared__ unsigned long long s_base;
    if (threadIdx.x < 32) {
        const unsigned long long base = tile_base_from_totals(p.tile_total, p.super_total, blockIdx.x);
        if (threadIdx.x == 0)
            s_base = base;
    }
    const uint64_t i = (uint64_t)blockIdx.x * RP_TILE + threadIdx.x;
    const bool pend = ev_pending(p, i);
    uint32_t tot;
    const uint32_t r = block_scan<uint32_t>(s_warp, pend ? 1u : 0u, &tot);
    if (pend) {
        const uint64_t k = s_base + r;
        p.item[k] = i;
        p.rec[k] = p.dir_rec ? p.dir_rec[i] : i;
        p.len[k] = p.dir_rec ? p.dir_len[i] : (uint32_t)(p.path_off[i + 1] - p.path_off[i]);
    }
    if (i + 1 == p.n)
        *p.count = s_base + tot;
}

/* ---- a subset stat read over the whole batch: every record reads as a node the batch owns at its payload length
   (SAME), then the subset's stats land on their records ---- */
struct EvStatFill {
    uint64_t n, m;
    const unsigned long long *json_off;
    long long want;
    const unsigned long long *rec;              /* [m] the subset's records */
    const int32_t *s_err, *s_ver, *s_dlen;      /* [m] */
    const long long *s_own;
    int32_t *err, *ver, *dlen;                  /* [n] */
    long long *own;
};

__global__ void __launch_bounds__(256) regk_events_stat_fill_kernel(const EvStatFill p)
{
    const uint64_t i = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= p.n)
        return;
    p.err[i] = 0;
    p.ver[i] = 0;
    p.own[i] = p.want;
    p.dlen[i] = (int32_t)(p.json_off[i + 1] - p.json_off[i]);
}

__global__ void __launch_bounds__(256) regk_events_stat_scatter_kernel(const EvStatFill p)
{
    const uint64_t k = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (k >= p.m)
        return;
    const uint64_t i = p.rec[k];
    p.err[i] = p.s_err[k];
    p.ver[i] = p.s_ver[k];
    p.own[i] = p.s_own[k];
    p.dlen[i] = p.s_dlen[k];
}

}  /* namespace regk */
#endif /* __CUDACC__ */
#endif /* REGK_EVENTS_CUH */
