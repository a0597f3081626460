/*
 * regk_stats.cuh — the heartbeat by stat: read ZooKeeper's ExistsResponse replies to the exists frames of a batch
 * (regk_jute_requests with REGK_ZK_EXISTS) and class the batch from the Stats alone.  The reference's heartbeat is one
 * zk.stat per node (lib/zk.js:21-44); no node data travels and none is compared.
 *
 * PARITY UNPINNED: the layout is restated from zookeeper.jute (ReplyHeader, ExistsResponse, Stat) and tested against an
 * independent restatement, not against a server.  A reply frame, big endian:
 *   int len | int xid | long zxid | int err | [ Stat (68 bytes) ]
 * The Stat is present iff err == 0, so len == 84 for a success and len == 16 for an error.  From the frame's first byte:
 *   czxid 20 | mzxid 28 | ctime 36 | mtime 44 | version 52 | cversion 56 | aversion 60 | ephemeralOwner 64 |
 *   dataLength 72 | numChildren 76 | pzxid 80
 * xid -1 (a watch notification) and -2 (a ping) are skipped whatever their body.
 *
 * stat_head() is the plausibility test of one position and stat_check() the full check of reply k; stat_mask16() is the
 * same plausibility test for the 16 start phases of one 16-byte block, from words held in registers.  All three are host
 * + device code (the CPU tests run them).
 *
 * reading   cand (stat_mask16() over every block at or after start: the success length is a constant, so the three words
 *           at +0, +4 and +16 decide a position), then regk_replies.cuh's compact, succ, jump and mark kernels and its
 *           chain count; the chain kernel here checks reply k < n against xid_base + k and writes err, version,
 *           ephemeralOwner, dataLength and mzxid per record.
 * classing  reply k answers record k, so there is no observed side: class (one thread per record: the class from its
 *           Stat, and its path into the table of first occurrences, regk_reconcile_desired_kernel's protocol), mark (DUP,
 *           match, the per-tile list counts), then regk_reconcile_compact_kernel and the gathers as every reconcile.
 */
#ifndef REGK_STATS_CUH
#define REGK_STATS_CUH

#include "regk_replies.cuh"

namespace regk {

/* stat_head / stat_check results */
enum : uint32_t {
    ST_OK = 0,
    ST_TRUNC,           /* the stream ends inside the frame (or before its length word) */
    ST_BAD_LEN,         /* len < 16: no room for a ReplyHeader */
    ST_NEG_XID,         /* a negative xid other than -1 / -2 */
    ST_XID_RANGE,       /* an xid outside [xid_base, xid_base + n) */
    ST_ERR_BODY,        /* err != 0 and a body */
    ST_SUCC_LEN,        /* err == 0 and len != 84 */
    ST_ORDER,           /* an xid in range but not xid_base + k */
    ST_NEG_DLEN,        /* Stat.dataLength < 0 */
};

constexpr int32_t ST_SUCC = 84;                 /* the length word of a success: ReplyHeader + Stat */

struct StatHead {
    uint32_t kind;      /* RK_* */
    int32_t len, xid, err;
};

/* the verdict on a position whose frame fits the stream, from its three words */
RG_HD uint32_t stat_words(int32_t L, int32_t xid, int32_t err, int32_t xid_base, uint64_t n)
{
    if (xid == -1 || xid == -2)
        return ST_OK;
    if ((uint64_t)((uint32_t)xid - (uint32_t)xid_base) >= n)
        return xid < 0 ? ST_NEG_XID : ST_XID_RANGE;
    if (err != 0)
        return L == 16 ? ST_OK : ST_ERR_BODY;
    return L == ST_SUCC ? ST_OK : ST_SUCC_LEN;
}

/* Plausibility of a frame starting at b, with `avail` stream bytes from b on (reads at most 20 of them, never past
   avail): the frame fits, its xid is -1, -2 or one of the n requests, an error has len 16 and a success len 84. */
RG_HD uint32_t stat_head(const uint8_t *b, uint64_t avail, int32_t xid_base, uint64_t n, StatHead *h)
{
    h->kind = RK_REPLY;
    h->len = h->xid = h->err = 0;
    if (avail < 4)
        return ST_TRUNC;
    const int32_t L = (int32_t)be32_at(b);
    h->len = L;
    if (L < 16)
        return ST_BAD_LEN;
    if ((uint64_t)L + 4u > avail)
        return ST_TRUNC;
    h->xid = (int32_t)be32_at(b + 4);
    h->err = (int32_t)be32_at(b + 16);
    if (h->xid == -1 || h->xid == -2)
        h->kind = h->xid == -1 ? RK_NOTIFY : RK_PING;
    return stat_words(L, h->xid, h->err, xid_base, n);
}

/* stat_head(), then the xid against xid_base + k and the Stat's dataLength.  Notifications and pings pass with their
   kind set. */
RG_HD uint32_t stat_check(const uint8_t *b, uint64_t avail, int32_t xid_base, uint64_t n, uint64_t k, StatHead *h)
{
    const uint32_t c = stat_head(b, avail, xid_base, n, h);
    if (c != ST_OK || h->kind != RK_REPLY)
        return c;
    if ((uint32_t)h->xid != (uint32_t)xid_base + (uint32_t)k)
        return ST_ORDER;
    if (h->err == 0 && (int32_t)be32_at(b + 72) < 0)
        return ST_NEG_DLEN;
    return ST_OK;
}

/* The big-endian word whose first byte is byte `sh` (0 .. 3) of the little-endian word lo; hi is the word after it.
   One byte permute on the device. */
RG_HD uint32_t st_be32(uint32_t lo, uint32_t hi, uint32_t sh)
{
#if defined(__CUDA_ARCH__)
    return __byte_perm(lo, hi, (sh + 3u) | (sh + 2u) << 4 | (sh + 1u) << 8 | sh << 12);
#else
    const uint32_t v = sh ? lo >> (8u * sh) | hi << (32u - 8u * sh) : lo;
    return v << 24 | (v & 0xFF00u) << 8 | (v >> 8 & 0xFF00u) | v >> 24;
#endif
}

/* stat_head() == ST_OK for the 16 positions of one 16-byte block, as a bit mask.  w[0 .. 8] = the block and the 20
   bytes after it as little-endian words (bytes at or past the stream's end read as anything); avail = stream bytes from
   the block's first byte on; positions below `first` are left out.  A position's frame fits iff len + 4 + f <= avail,
   which also keeps its three words inside the stream. */
RG_HD uint32_t stat_mask16(const uint32_t *w, uint64_t avail, uint32_t first, int32_t xid_base, uint64_t n)
{
    const uint32_t room = avail > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)avail;     /* len + 4 + f < 2^31 + 20 */
    uint32_t mask = 0;
#if defined(__CUDA_ARCH__)
    #pragma unroll
#endif
    for (uint32_t f = 0; f < 16u; f++) {
        const uint32_t q = f >> 2, sh = f & 3u;
        const int32_t L = (int32_t)st_be32(w[q], w[q + 1], sh);
        const int32_t xid = (int32_t)st_be32(w[q + 1], w[q + 2], sh);
        const int32_t err = (int32_t)st_be32(w[q + 4], w[q + 5], sh);
        const bool fits = f >= first && L >= 16 && (uint32_t)L + 4u + f <= room;
        if (fits && stat_words(L, xid, err, xid_base, n) == ST_OK)
            mask |= 1u << f;
    }
    return mask;
}

}  /* namespace regk */

#if defined(__CUDACC__)
#include "regk_reconcile.cuh"

namespace regk {

struct StatParams {
    RepParams r;                                /* the frame chain: r.n = records, r.err / r.ver / r.own per record */
    uint64_t start;
    unsigned long long *fpos;                   /* [n] the reply's position */
    int32_t *dlen;                              /* [n] Stat.dataLength */
    long long *mzxid;                           /* [n] Stat.mzxid */
};

/* ---- cand: the plausible positions at or after start, 16 per thread, tested from registers ---- */
__global__ void __launch_bounds__(RP_TILE) regk_stats_cand_kernel(const StatParams sp)
{
    const RepParams &p = sp.r;
    __shared__ uint32_t s_warp[WARPS];
    const uint64_t nblk = (p.len + 15u) / 16u;
    const uint64_t b = (uint64_t)blockIdx.x * RP_TILE + threadIdx.x;
    uint32_t mask = 0;
    if (b < nblk && 16ull * b + 16u > sp.start) {
        const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
        const uint4 v0 = rp_block(p.s, p.len, b);
        const uint4 v1 = b + 1 < nblk ? rp_block(p.s, p.len, b + 1) : zero;
        const uint4 v2 = b + 2 < nblk ? rp_block(p.s, p.len, b + 2) : zero;
        const uint32_t w[9] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w, v2.x};
        const uint64_t at = 16ull * b;
        mask = stat_mask16(w, p.len - at, sp.start > at ? (uint32_t)(sp.start - at) : 0u, p.xid_base, p.n);
    }
    uint32_t total;
    const uint32_t rank = block_scan<uint32_t>(s_warp, (uint32_t)__popc(mask), &total);
    if (b < nblk)
        p.word[b] = mask | rank << 16;
    if (threadIdx.x == 0)
        add_tile_total(p.tile_total, p.super_total, blockIdx.x, total);
}

/* ---- cand, the form of regk_replies_cand_kernel: stat_head() on bytes staged in shared memory.  Kept for the A/B
   measurement of the register form (option "stats_cand_shared"); same output. ---- */
__global__ void __launch_bounds__(RP_TILE) regk_stats_cand_shared_kernel(const StatParams sp)
{
    const RepParams &p = sp.r;
    __shared__ __align__(16) uint8_t s_win[RP_SPAN + 32];
    __shared__ uint32_t s_warp[WARPS];
    const uint64_t nblk = (p.len + 15u) / 16u;
    const uint64_t b0 = (uint64_t)blockIdx.x * RP_TILE, b = b0 + threadIdx.x;
    const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
    reinterpret_cast<uint4 *>(s_win)[threadIdx.x] = b < nblk ? rp_block(p.s, p.len, b) : zero;
    if (threadIdx.x < 2) {
        const uint64_t e = b0 + RP_TILE + threadIdx.x;
        reinterpret_cast<uint4 *>(s_win)[RP_TILE + threadIdx.x] = e < nblk ? rp_block(p.s, p.len, e) : zero;
    }
    __syncthreads();
    uint32_t mask = 0;
    if (b < nblk && 16ull * b + 16u > sp.start) {
        for (uint32_t f = 0; f < 16u; f++) {
            const uint64_t pos = 16ull * b + f;
            if (pos >= p.len)
                break;
            StatHead h;
            if (pos >= sp.start && stat_head(s_win + 16u * threadIdx.x + f, p.len - pos, p.xid_base, p.n, &h) == ST_OK)
                mask |= 1u << f;
        }
    }
    uint32_t total;
    const uint32_t rank = block_scan<uint32_t>(s_warp, (uint32_t)__popc(mask), &total);
    if (b < nblk)
        p.word[b] = mask | rank << 16;
    if (threadIdx.x == 0)
        add_tile_total(p.tile_total, p.super_total, blockIdx.x, total);
}

RG_HD long long st_be64_at(const uint8_t *b)
{
    return (long long)((unsigned long long)be32_at(b) << 32 | be32_at(b + 4));
}

/* ---- chain: k of every reply frame, the check of k < n, the per-record arrays and the found / missing / other counts ---- */
__global__ void __launch_bounds__(RP_TILE) regk_stats_chain_kernel(const StatParams sp)
{
    const RepParams &p = sp.r;
    __shared__ uint32_t s_warp[WARPS];
    __shared__ unsigned long long s_base;
    __shared__ uint32_t s_cnt[4];                   /* skipped, found, missing, other errors */
    if (threadIdx.x < 4)
        s_cnt[threadIdx.x] = 0;
    if (threadIdx.x < 32) {
        const unsigned long long base = tile_base_from_totals(p.tile_total, p.super_total, blockIdx.x);
        if (threadIdx.x == 0)
            s_base = base;
    }
    const uint64_t c = (uint64_t)blockIdx.x * RP_TILE + threadIdx.x;
    const bool on = c < p.C && p.marked[c];
    const bool rep = rp_is_reply(p, c);
    uint32_t tot;
    const uint32_t r = block_scan<uint32_t>(s_warp, rep ? 1u : 0u, &tot);      /* its barriers publish s_base, s_cnt */
    const uint64_t k = s_base + r;
    if (on && k < p.n) {
        if (!rep) {
            atomicAdd(&s_cnt[0], 1u);
        } else {
            const unsigned long long pos = p.cand[c];
            const uint8_t *fr = p.s + pos;
            StatHead h;
            const uint32_t code = stat_check(fr, p.len - pos, p.xid_base, p.n, k, &h);
            sp.fpos[k] = pos;
            if (code != ST_OK) {
                atomicMin(p.counters + RQ_ERR, (unsigned long long)k << 8 | code);
            } else {
                const bool found = h.err == 0;      /* a record without a node reads as zeros */
                p.err[k] = h.err;
                p.ver[k] = found ? (int32_t)be32_at(fr + 52) : 0;
                p.own[k] = found ? st_be64_at(fr + 64) : 0ll;
                sp.dlen[k] = found ? (int32_t)be32_at(fr + 72) : 0;
                sp.mzxid[k] = found ? st_be64_at(fr + 28) : 0ll;
                atomicAdd(&s_cnt[found ? 1 : h.err == -101 ? 2 : 3], 1u);
                if (k + 1 == p.n)
                    p.counters[RQ_CONSUMED] = pos + 4u + (uint32_t)h.len;
            }
        }
    }
    if (c + 1 == p.C)
        p.counters[RQ_NREP] = s_base + tot;
    __syncthreads();
    if (threadIdx.x < 4 && s_cnt[threadIdx.x])
        atomicAdd(p.counters + (threadIdx.x == 0 ? RQ_SKIP : RQ_FOUND + threadIdx.x - 1), (unsigned long long)s_cnt[threadIdx.x]);
}

/* What regk_reconcile_stats classes from: the per-record arrays of the last read, and ReconcileParams for everything
   the reconcile passes share (rc.m == 0: there is no observed side). */
struct StatClassParams {
    ReconcileParams rc;
    const int32_t *err;                         /* [n] */
    const long long *own;
    const int32_t *dlen;
    const long long *mzxid;
    const long long *known_mzxid;               /* [n] or NULL */
};

/* ---- class: the record's class from its Stat; its path into T_d, the first record keeps the slot.  A reply with an
   error other than NONODE is reported as the smallest such record (counters[RC_C_BAD]). ---- */
__global__ void __launch_bounds__(256, 4) regk_stats_class_kernel(const StatClassParams sp)
{
    const ReconcileParams &p = sp.rc;
    const uint64_t i = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= p.n)
        return;
    const int32_t e = sp.err[i];
    uint8_t c = RC_CREATE;
    if (e == 0) {
        const uint32_t jl = (uint32_t)(p.d_json_off[i + 1] - p.d_json_off[i]);
        c = sp.own[i] != p.want ? RC_REPLACE
          : (uint32_t)sp.dlen[i] != jl || (sp.known_mzxid && sp.mzxid[i] != sp.known_mzxid[i]) ? RC_UPDATE : RC_SAME;
    } else if (e != -101) {
        atomicMin(p.counters + RC_C_BAD, (unsigned long long)i);
    }
    p.cls[i] = c;
    const unsigned long long o0 = p.d_path_off[i];
    const uint32_t len = (uint32_t)(p.d_path_off[i + 1] - o0);
    const uint32_t *W = reinterpret_cast<const uint32_t *>(p.d_path);
    uint32_t slot = string_hash32(W, o0, len) & p.mask_d;
    for (;;) {
        uint32_t cur = p.t_des[slot];
        if (cur == 0u) {
            cur = atomicCAS(p.t_des + slot, 0u, (uint32_t)i + 1u);
            if (cur == 0u)
                break;
        }
        const uint64_t k = cur - 1u;
        if (k == i)
            break;
        const unsigned long long k0 = p.d_path_off[k];
        if ((uint32_t)(p.d_path_off[k + 1] - k0) == len && string_equal(W, o0, k0, len)) {
            if (cur > (uint32_t)i + 1u)
                atomicMin(p.t_des + slot, (uint32_t)i + 1u);
            break;
        }
        slot = (slot + 1u) & p.mask_d;
    }
    p.slot_des[i] = slot;
}

/* ---- mark: DUP records, match (the first record with the path, ~0 when its node is missing), per-tile list counts ---- */
__global__ void __launch_bounds__(RC_TILE) regk_stats_mark_kernel(const StatClassParams sp)
{
    const ReconcileParams &p = sp.rc;
    const uint64_t i = (uint64_t)blockIdx.x * RC_TILE + threadIdx.x;
    uint32_t f = 0;                                         /* bit k: goes to list k */
    if (i < p.n) {
        uint8_t c = p.cls[i];
        const uint64_t first = p.t_des[p.slot_des[i]] - 1u;
        if (first != i) {
            c = RC_DUP;
            p.cls[i] = c;
        }
        p.match[i] = sp.err[first] == 0 ? first : ~0ull;
        f = c == RC_CREATE ? 1u << RC_LCREATE : c == RC_UPDATE ? 1u << RC_LUPDATE : c == RC_DUP ? 1u << RC_LDUP :
            c == RC_REPLACE ? 1u << RC_LREPLACE : 0u;
    }
    #pragma unroll
    for (int l = RC_LCREATE; l < RC_NREC_LISTS; l++) {
        const uint32_t c = __popc(__ballot_sync(0xFFFFFFFFu, (f >> l) & 1u));
        if ((threadIdx.x & 31u) == 0)
            add_tile_total(p.tile_total[l], p.super_total[l], blockIdx.x, c);
    }
}

}  /* namespace regk */
#endif /* __CUDACC__ */
#endif /* REGK_STATS_CUH */
