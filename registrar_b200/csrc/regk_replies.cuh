/*
 * regk_replies.cuh — read ZooKeeper's GetDataResponse replies to the getData frames of a batch (regk_jute_requests with
 * REGK_ZK_GETDATA) and turn them into the snapshot regk_reconcile_owned takes: one node per distinct path among the
 * found replies, with its data, Stat.version and Stat.ephemeralOwner.  The batch form of the reference's heartbeat,
 * which stats every node (lib/zk.js:21-44, lib/index.js:131-159).
 *
 * A reply frame, big endian (zookeeper.jute ReplyHeader, GetDataResponse, Stat):
 *   int len | int xid | long zxid | int err | [ buffer data (int D, D bytes; D = -1: null) | Stat (68 bytes) ]
 * The body is present iff err == 0, so len == 16 for an error and len == 88 + max(D, 0) for a success.  The Stat is
 *   czxid mzxid ctime mtime (8 each) | version cversion aversion (4 each) | ephemeralOwner (8) | dataLength numChildren
 *   (4 each) | pzxid (8)
 * so, from the frame's first byte, D sits at 20, the data at 24, version at 56 + max(D, 0), ephemeralOwner at 68 + ...,
 * dataLength at 76 + ....  xid -1 (a watch notification) and -2 (a ping) are skipped whatever their body.
 *
 * reply_head() is the plausibility test of one position and reply_check() the full per-frame check; both are host +
 * device code (the CPU tests run them, and the library runs reply_head() on the host once, where a chain stops).
 *
 * The stream is a chain: each frame's length says where the next starts, and no thread walks it.  The passes:
 *   cand      every byte position at once: a CTA stages 2 KB of the stream (+ 32 bytes) in shared memory, each thread
 *             tests the 16 start phases of one 16-byte block with reply_head() and writes a word per block: the 16-bit
 *             candidate mask and, above it, the block's candidate rank inside the CTA.  Per-CTA counts go into
 *             two-level totals.
 *   compact   the candidates' positions in position order; each CTA's first rank goes to tile_base[].
 *   succ      J_0(c) = the candidate at p_c + 4 + len_c, by rank (tile_base + the block's rank + a popcount), or none.
 *   jump      J_{l+1}(c) = J_l(J_l(c)), l = 0 .. K - 1, with 2^(K+1) >= the number of candidates.
 *   mark      from K down to 0: every marked c marks J_l(c); position 0 seeds it.  The marked set is exactly the chain
 *             from 0 (marks made within a level are chain frames too, so the race is harmless).  A candidate inside
 *             node data that looks like a frame is never reached.
 *   chain     the chain's reply frames get k (a scan over the marked candidates that are not notifications or pings);
 *             reply k < n is checked with reply_check() against xid_base + k, and its err, data position, data length,
 *             version and owner land in per-record arrays.  The smallest failing k is kept (k << 8 | code).
 *   insert    found records into an open-addressing table keyed by their path in the batch (the protocol of
 *             regk_reconcile_desired_kernel: atomicCAS claims a slot, paths compared byte for byte, atomicMin keeps the
 *             first record).
 *   nodes     records that are found and own their slot become nodes, in record order, with their stats and lengths.
 * regk_mkdirp_len_kernel / regk_mkdirp_gather_kernel then pack the node paths (from the batch) and data (from the stream).
 */
#ifndef REGK_REPLIES_CUH
#define REGK_REPLIES_CUH

#include "regk_core.cuh"

namespace regk {

/* reply_head / reply_check results: RP_OK, or why the frame at that position cannot be the next reply */
enum : uint32_t {
    RP_OK = 0,
    RP_TRUNC,           /* the stream ends inside the frame (or before its length word) */
    RP_BAD_LEN,         /* len < 16: no room for a ReplyHeader */
    RP_NEG_XID,         /* a negative xid other than -1 / -2 */
    RP_XID_RANGE,       /* an xid outside [xid_base, xid_base + n) */
    RP_ERR_BODY,        /* err != 0 and a body */
    RP_SUCC_LEN,        /* err == 0 and len != 88 + max(D, 0) */
    RP_NEG_DATA,        /* D < -1 */
    RP_STAT_LEN,        /* Stat.dataLength != max(D, 0) */
    RP_ORDER,           /* an xid in range but not xid_base + k: out of order, or a record that already has a reply */
};
enum : uint32_t { RK_REPLY = 0, RK_NOTIFY = 1, RK_PING = 2 };

struct ReplyHead {
    uint32_t kind;      /* RK_* */
    int32_t len, xid, err;
    int32_t dlen;       /* D of a success frame, else 0 */
};

RG_HD uint32_t be32_at(const uint8_t *b)
{
    return (uint32_t)b[0] << 24 | (uint32_t)b[1] << 16 | (uint32_t)b[2] << 8 | (uint32_t)b[3];
}

/* Plausibility of a frame starting at b, with `avail` stream bytes from b on (reads at most 24 of them, never past
   avail): the frame fits, its xid is -1, -2 or one of the n requests, and an in-range reply has the length its err and
   data length call for. */
RG_HD uint32_t reply_head(const uint8_t *b, uint64_t avail, int32_t xid_base, uint64_t n, ReplyHead *h)
{
    h->kind = RK_REPLY;
    h->len = h->xid = h->err = h->dlen = 0;
    if (avail < 4)
        return RP_TRUNC;
    const int32_t L = (int32_t)be32_at(b);
    h->len = L;
    if (L < 16)
        return RP_BAD_LEN;
    if ((uint64_t)L + 4u > avail)
        return RP_TRUNC;
    const int32_t xid = (int32_t)be32_at(b + 4), err = (int32_t)be32_at(b + 16);
    h->xid = xid;
    h->err = err;
    if (xid == -1 || xid == -2) {
        h->kind = xid == -1 ? RK_NOTIFY : RK_PING;
        return RP_OK;
    }
    if ((uint64_t)((uint32_t)xid - (uint32_t)xid_base) >= n)
        return xid < 0 ? RP_NEG_XID : RP_XID_RANGE;
    if (err != 0)
        return L == 16 ? RP_OK : RP_ERR_BODY;
    if (L < 20)                                 /* no room for D */
        return RP_SUCC_LEN;
    const int32_t D = (int32_t)be32_at(b + 20);
    h->dlen = D;
    if (D < -1)
        return RP_NEG_DATA;
    if ((int64_t)L != 88 + (int64_t)(D > 0 ? D : 0))
        return RP_SUCC_LEN;
    return RP_OK;
}

/* The full check of the frame at b as the reply to record k: reply_head(), then its xid against xid_base + k and the
   Stat's dataLength against the data it carries.  Notifications and pings pass with their kind set. */
RG_HD uint32_t reply_check(const uint8_t *b, uint64_t avail, int32_t xid_base, uint64_t n, uint64_t k, ReplyHead *h)
{
    const uint32_t c = reply_head(b, avail, xid_base, n, h);
    if (c != RP_OK || h->kind != RK_REPLY)
        return c;
    if ((uint32_t)h->xid != (uint32_t)xid_base + (uint32_t)k)
        return RP_ORDER;
    if (h->err == 0) {
        const uint32_t dp = h->dlen > 0 ? (uint32_t)h->dlen : 0u;
        if (be32_at(b + 76 + dp) != dp)
            return RP_STAT_LEN;
    }
    return RP_OK;
}

}  /* namespace regk */

#if defined(__CUDACC__)
#include "regk_kernels.cuh"

namespace regk {

constexpr uint32_t RP_TILE = TILE;              /* threads per CTA of the block-scanned passes (128) */
constexpr uint32_t RP_SPAN = RP_TILE * 16u;     /* stream bytes per candidate CTA */
constexpr uint32_t RP_NONE = 0xFFFFFFFFu;       /* no successor / no slot */

/* counters[] */
enum { RQ_ERR = 0, RQ_NREP, RQ_SKIP, RQ_FOUND, RQ_MISSING, RQ_ERROR, RQ_CONSUMED, RQ_M, RQ_STOP, RQ_NCOUNTERS };

struct RepParams {
    const uint8_t *s;                           /* the reply stream (device) */
    uint64_t len;
    int32_t xid_base;
    uint64_t n;                                 /* records of the framed batch */
    uint32_t *word;                             /* [blocks] candidate mask | in-CTA rank << 16 */
    uint32_t *tile_total;                       /* two-level totals of the pass running (reset between passes) */
    unsigned long long *super_total;
    unsigned long long *tile_base;              /* [cand CTAs] rank of each CTA's first candidate */
    unsigned long long *cand;                   /* [C] candidate positions, ascending */
    uint64_t C;
    uint8_t *marked;                            /* [C] on the chain from position 0 */
    /* per record k < n */
    int32_t *err;
    unsigned long long *data_pos;               /* stream position of the reply's data */
    uint32_t *dlen;                             /* max(D, 0) */
    int32_t *ver;
    long long *own;
    uint32_t *slot;                             /* table slot of a found record, RP_NONE otherwise */
    /* the batch's path stream (>= 16 bytes of slack) and the dedup table */
    const uint8_t *d_path;
    const unsigned long long *d_path_off;
    uint32_t *table;                            /* record + 1, 0 = empty (zeroed by the host) */
    uint32_t mask_t;
    /* per node j < m */
    unsigned long long *node_rec;
    int32_t *node_ver;
    long long *node_own;
    uint32_t *node_plen, *node_dlen;
    unsigned long long *counters;               /* [RQ_NCOUNTERS] */
};

__device__ __forceinline__ uint4 rp_block(const uint8_t *s, uint64_t len, uint64_t blk)
{
    const uint64_t a = 16ull * blk;
    if (a + 16u <= len)
        return __ldg(reinterpret_cast<const uint4 *>(s + a));
    uint32_t w[4] = {0u, 0u, 0u, 0u};           /* the stream's last, partial block: never a byte at or past len */
    #pragma unroll
    for (uint32_t k = 0; k < 16u; k++)
        if (a + k < len)
            w[k >> 2] |= (uint32_t)s[a + k] << (8u * (k & 3u));
    return make_uint4(w[0], w[1], w[2], w[3]);
}

/* ---- cand: the plausible positions of 16 x 128 bytes ---- */
__global__ void __launch_bounds__(RP_TILE) regk_replies_cand_kernel(const RepParams p)
{
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
    if (b < nblk) {
        for (uint32_t f = 0; f < 16u; f++) {
            const uint64_t pos = 16ull * b + f;
            if (pos >= p.len)
                break;
            ReplyHead h;
            if (reply_head(s_win + 16u * threadIdx.x + f, p.len - pos, p.xid_base, p.n, &h) == RP_OK)
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

/* ---- compact: candidate positions in order, each CTA's base ---- */
__global__ void __launch_bounds__(RP_TILE) regk_replies_compact_kernel(const RepParams p)
{
    __shared__ unsigned long long s_base;
    if (threadIdx.x < 32) {
        const unsigned long long base = tile_base_from_totals(p.tile_total, p.super_total, blockIdx.x);
        if (threadIdx.x == 0) {
            s_base = base;
            p.tile_base[blockIdx.x] = base;
        }
    }
    __syncthreads();
    const uint64_t nblk = (p.len + 15u) / 16u;
    const uint64_t b = (uint64_t)blockIdx.x * RP_TILE + threadIdx.x;
    if (b < nblk) {
        const uint32_t w = p.word[b];
        uint32_t m = w & 0xFFFFu;
        unsigned long long r = s_base + (w >> 16);
        while (m) {
            p.cand[r++] = 16ull * b + (uint32_t)(__ffs(m) - 1);
            m &= m - 1u;
        }
    }
}

/* ---- succ: J_0 ---- */
__global__ void __launch_bounds__(256) regk_replies_succ_kernel(const RepParams p, uint32_t *j0)
{
    const uint64_t c = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (c >= p.C)
        return;
    const unsigned long long pos = p.cand[c];
    const unsigned long long q = pos + 4u + be32_at(p.s + pos);   /* a candidate's frame fits: q <= len */
    uint32_t nx = RP_NONE;
    if (q < p.len) {
        const uint32_t w = p.word[q >> 4], f = (uint32_t)(q & 15u);
        if ((w >> f) & 1u)
            nx = (uint32_t)(p.tile_base[q / RP_SPAN] + (w >> 16) + (uint32_t)__popc(w & ((1u << f) - 1u)));
    }
    j0[c] = nx;
}

/* ---- jump: J_{l+1} = J_l o J_l ---- */
__global__ void __launch_bounds__(256) regk_replies_jump_kernel(const uint32_t *__restrict__ jin, uint32_t *__restrict__ jout,
    uint64_t C)
{
    const uint64_t c = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (c >= C)
        return;
    const uint32_t a = jin[c];
    jout[c] = a == RP_NONE ? RP_NONE : jin[a];
}

/* ---- mark: one level; `seed` (the top level) marks position 0's candidate first ---- */
__global__ void __launch_bounds__(256) regk_replies_mark_kernel(const RepParams p, const uint32_t *__restrict__ jl, uint32_t seed)
{
    const uint64_t c = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (c >= p.C)
        return;
    bool m = p.marked[c] != 0;
    if (seed && c == 0 && p.cand[0] == 0) {
        p.marked[0] = 1;
        m = true;
    }
    if (m) {
        const uint32_t j = jl[c];
        if (j != RP_NONE)
            p.marked[j] = 1;
    }
}

/* ---- chain: count the chain's reply frames per CTA ---- */
__device__ __forceinline__ bool rp_is_reply(const RepParams &p, uint64_t c)
{
    if (c >= p.C || !p.marked[c])
        return false;
    const int32_t xid = (int32_t)be32_at(p.s + p.cand[c] + 4);
    return xid != -1 && xid != -2;
}

__global__ void __launch_bounds__(RP_TILE) regk_replies_chain_count_kernel(const RepParams p)
{
    const uint64_t c = (uint64_t)blockIdx.x * RP_TILE + threadIdx.x;
    const uint32_t cnt = (uint32_t)__popc(__ballot_sync(0xFFFFFFFFu, rp_is_reply(p, c)));
    if ((threadIdx.x & 31u) == 0)
        add_tile_total(p.tile_total, p.super_total, blockIdx.x, cnt);
}

/* ---- chain: k of every reply frame, the full check of k < n, the per-record arrays ---- */
__global__ void __launch_bounds__(RP_TILE) regk_replies_chain_kernel(const RepParams p)
{
    __shared__ uint32_t s_warp[WARPS];
    __shared__ unsigned long long s_base;
    __shared__ uint32_t s_skip;
    if (threadIdx.x < 32) {
        const unsigned long long base = tile_base_from_totals(p.tile_total, p.super_total, blockIdx.x);
        if (threadIdx.x == 0) {
            s_base = base;
            s_skip = 0;
        }
    }
    const uint64_t c = (uint64_t)blockIdx.x * RP_TILE + threadIdx.x;
    const bool on = c < p.C && p.marked[c];
    const bool rep = rp_is_reply(p, c);
    uint32_t tot;
    const uint32_t r = block_scan<uint32_t>(s_warp, rep ? 1u : 0u, &tot);      /* its barriers publish s_base */
    const uint64_t k = s_base + r;                  /* replies before this frame */
    if (on && k < p.n) {
        if (!rep) {
            atomicAdd(&s_skip, 1u);
        } else {
            const unsigned long long pos = p.cand[c];
            ReplyHead h;
            const uint32_t code = reply_check(p.s + pos, p.len - pos, p.xid_base, p.n, k, &h);
            p.data_pos[k] = pos + 24u;                  /* also names the frame of a refusal */
            if (code != RP_OK) {
                atomicMin(p.counters + RQ_ERR, (unsigned long long)k << 8 | code);
            } else {
                const uint32_t dp = h.err == 0 && h.dlen > 0 ? (uint32_t)h.dlen : 0u;
                p.err[k] = h.err;
                p.dlen[k] = dp;
                if (h.err == 0) {
                    const uint8_t *st = p.s + pos + 24u + dp;
                    p.ver[k] = (int32_t)be32_at(st + 32);
                    p.own[k] = (long long)((unsigned long long)be32_at(st + 44) << 32 | be32_at(st + 48));
                }
                if (k + 1 == p.n)
                    p.counters[RQ_CONSUMED] = pos + 4u + (uint32_t)h.len;
            }
        }
    }
    if (c + 1 == p.C)
        p.counters[RQ_NREP] = s_base + tot;
    __syncthreads();
    if (threadIdx.x == 0 && s_skip)
        atomicAdd(p.counters + RQ_SKIP, (unsigned long long)s_skip);
}

/* ---- the end of the chain, when it holds fewer than n replies: the largest marked frame end ---- */
__global__ void __launch_bounds__(256) regk_replies_stop_kernel(const RepParams p)
{
    const uint64_t c = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (c < p.C && p.marked[c]) {
        const unsigned long long pos = p.cand[c];
        atomicMax(p.counters + RQ_STOP, pos + 4u + be32_at(p.s + pos));
    }
}

/* ---- insert: found records into the table, keyed by their path in the batch; the first record keeps the slot.
   (256, 4) as the reconcile passes with the same loop. ---- */
__global__ void __launch_bounds__(256, 4) regk_replies_insert_kernel(const RepParams p)
{
    const uint64_t i = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= p.n)
        return;
    if (p.err[i] != 0) {
        p.slot[i] = RP_NONE;
        return;
    }
    const unsigned long long o0 = p.d_path_off[i];
    const uint32_t len = (uint32_t)(p.d_path_off[i + 1] - o0);
    const uint32_t *W = reinterpret_cast<const uint32_t *>(p.d_path);
    uint32_t slot = string_hash32(W, o0, len) & p.mask_t;
    for (;;) {
        uint32_t cur = p.table[slot];
        if (cur == 0u) {
            cur = atomicCAS(p.table + slot, 0u, (uint32_t)i + 1u);
            if (cur == 0u)
                break;
        }
        const uint64_t k = cur - 1u;
        if (k == i)
            break;
        const unsigned long long k0 = p.d_path_off[k];
        if ((uint32_t)(p.d_path_off[k + 1] - k0) == len && string_equal(W, o0, k0, len)) {
            if (cur > (uint32_t)i + 1u)
                atomicMin(p.table + slot, (uint32_t)i + 1u);
            break;
        }
        slot = (slot + 1u) & p.mask_t;
    }
    p.slot[i] = slot;
}

/* ---- nodes: per-CTA counts of the records that become nodes, and of found / missing / other replies ---- */
__device__ __forceinline__ bool rp_is_node(const RepParams &p, uint64_t i)
{
    return i < p.n && p.slot[i] != RP_NONE && p.table[p.slot[i]] == (uint32_t)i + 1u;
}

__global__ void __launch_bounds__(RP_TILE) regk_replies_node_count_kernel(const RepParams p)
{
    __shared__ uint32_t s_cnt[3];
    if (threadIdx.x < 3)
        s_cnt[threadIdx.x] = 0;
    __syncthreads();
    const uint64_t i = (uint64_t)blockIdx.x * RP_TILE + threadIdx.x;
    const uint32_t cnt = (uint32_t)__popc(__ballot_sync(0xFFFFFFFFu, rp_is_node(p, i)));
    if ((threadIdx.x & 31u) == 0)
        add_tile_total(p.tile_total, p.super_total, blockIdx.x, cnt);
    if (i < p.n) {
        const int32_t e = p.err[i];
        atomicAdd(&s_cnt[e == 0 ? 0 : e == -101 ? 1 : 2], 1u);
    }
    __syncthreads();
    if (threadIdx.x < 3 && s_cnt[threadIdx.x])
        atomicAdd(p.counters + RQ_FOUND + threadIdx.x, (unsigned long long)s_cnt[threadIdx.x]);
}

__global__ void __launch_bounds__(RP_TILE) regk_replies_node_kernel(const RepParams p)
{
    __shared__ uint32_t s_warp[WARPS];
    __shared__ unsigned long long s_base;
    if (threadIdx.x < 32) {
        const unsigned long long base = tile_base_from_totals(p.tile_total, p.super_total, blockIdx.x);
        if (threadIdx.x == 0)
            s_base = base;
    }
    const uint64_t i = (uint64_t)blockIdx.x * RP_TILE + threadIdx.x;
    const bool node = rp_is_node(p, i);
    uint32_t tot;
    const uint32_t r = block_scan<uint32_t>(s_warp, node ? 1u : 0u, &tot);
    if (node) {
        const uint64_t j = s_base + r;
        p.node_rec[j] = i;
        p.node_ver[j] = p.ver[i];
        p.node_own[j] = p.own[i];
        p.node_plen[j] = (uint32_t)(p.d_path_off[i + 1] - p.d_path_off[i]);
        p.node_dlen[j] = p.dlen[i];
    }
    if (i + 1 == p.n)
        p.counters[RQ_M] = s_base + tot;
}

}  /* namespace regk */
#endif /* __CUDACC__ */
#endif /* REGK_REPLIES_CUH */
