/*
 * regk_children.cuh — list a batch's service directories with getChildren and class every child: the instances the
 * batch produces (and the directories on the way to them) are kept, every other child is stale.  The reference only
 * removes a node through its own unregister (lib/register.js:254-295) or through session expiry, which keeps a dead
 * instance in DNS for minutes (README.md:70-76, :764-779); a registrar that keeps a whole fleet registered can delete
 * such nodes at once when it knows which children of its service directories it did not produce.
 *
 * A reply frame, big endian (zookeeper.jute ReplyHeader, GetChildrenResponse):
 *   int len | int xid | long zxid | int err | [ int count | count x (int L | L bytes) ]
 * The body is present iff err == 0, so len == 16 for an error and len == 20 + sum(4 + L_i) for a success; count == -1
 * (a null vector) reads as no children.  xid -1 (a watch notification) and -2 (a ping) are skipped whatever their body.
 *
 * children_head() is the plausibility test of one position, children_check() the frame check of reply k and
 * children_entry() the check of one listing entry; all three are host + device code (the CPU tests run them).
 *
 * No thread walks the stream, and no thread walks a directory's entries one by one.  The passes:
 *   frames   the frame chain of regk_replies.cuh from position `start`: cand (children_head() at every position at
 *            or after start), then regk_replies.cuh's compact, succ, jump and mark kernels; the chain's replies get k
 *            by a scan (regk_replies_chain_count_kernel + the chain kernel here), and reply k < d is checked against
 *            xid_base + k.  Its position, end, err and entry count land in per-directory arrays.
 *   entries  the same machinery once more, inside the reached success frames: every position q of a frame body with
 *            room for a length word L >= 1 and L name bytes before the frame's end, whose first name byte is neither
 *            NUL nor '/', is a candidate; its successor is q + 4 + L.  A frame's end is the next frame's start, never
 *            a candidate, so chains never cross frames; each frame seeds its chain at its first entry (+24), and the
 *            jump tables need 2^(K+1) > the largest count, not the total.  The marked entries, ranked by a scan, are
 *            the children in stream order; each frame then compares its chain with its count (ent_frame kernel):
 *            the first failing entry, a count larger than the chain, or entries that end before the frame does.
 *   listing  path e = directory + '/' + name: lengths, regk_mkdirp_len_kernel's totals, and an output-stationary
 *            gather from the packed directories and the reply stream.
 *   keep     one open-addressing table of 64-bit slots ((record + 1) << 32 | length) holds the batch's paths and
 *            every prefix of every listed directory that ends at a component boundary (its mkdirp closure); a slot
 *            is claimed by atomicCAS, bytes are compared byte for byte, a hash only picks the slot.  Each listing
 *            path probes it: found = KEEP, else STALE.
 *   stale    compacted in listing order; regk_mkdirp_len_kernel / regk_mkdirp_gather_kernel pack their paths for the
 *            delete framing.
 */
#ifndef REGK_CHILDREN_CUH
#define REGK_CHILDREN_CUH

#include "regk_replies.cuh"

namespace regk {

/* children_head / children_check / children_entry results */
enum : uint32_t {
    CH_OK = 0,
    CH_TRUNC,           /* the stream ends inside the frame (or before its length word) */
    CH_BAD_LEN,         /* len < 16: no room for a ReplyHeader */
    CH_NEG_XID,         /* a negative xid other than -1 / -2 */
    CH_XID_RANGE,       /* an xid outside [xid_base, xid_base + d) */
    CH_ERR_BODY,        /* err != 0 and a body */
    CH_SUCC_LEN,        /* err == 0 and len < 20, or too short for count entries of 5 bytes or more */
    CH_NEG_COUNT,       /* count < -1 */
    CH_ORDER,           /* an xid in range but not xid_base + k */
    CH_ENT_TRUNC,       /* an entry (its length word or its name) runs past the frame's end */
    CH_ENT_EMPTY,       /* an entry with L < 1 */
    CH_NAME_SLASH,      /* a name holding '/' */
    CH_NAME_NUL,        /* a name holding a NUL byte */
    CH_NAME_DOT,        /* a name that is "." or ".." */
    CH_ENT_END,         /* the count's entries end before the frame does */
};

struct ChildHead {
    uint32_t kind;      /* RK_* */
    int32_t len, xid, err;
    int32_t count;      /* the vector's count of a success frame, else 0 */
};

/* Plausibility of a frame starting at b, with `avail` stream bytes from b on (reads at most 24 of them, never past
   avail): the frame fits, its xid is -1, -2 or one of the d requests, an in-range error has len 16, and a success
   has room for its count and for count entries of at least 5 bytes. */
RG_HD uint32_t children_head(const uint8_t *b, uint64_t avail, int32_t xid_base, uint64_t d, ChildHead *h)
{
    h->kind = RK_REPLY;
    h->len = h->xid = h->err = h->count = 0;
    if (avail < 4)
        return CH_TRUNC;
    const int32_t L = (int32_t)be32_at(b);
    h->len = L;
    if (L < 16)
        return CH_BAD_LEN;
    if ((uint64_t)L + 4u > avail)
        return CH_TRUNC;
    const int32_t xid = (int32_t)be32_at(b + 4), err = (int32_t)be32_at(b + 16);
    h->xid = xid;
    h->err = err;
    if (xid == -1 || xid == -2) {
        h->kind = xid == -1 ? RK_NOTIFY : RK_PING;
        return CH_OK;
    }
    if ((uint64_t)((uint32_t)xid - (uint32_t)xid_base) >= d)
        return xid < 0 ? CH_NEG_XID : CH_XID_RANGE;
    if (err != 0)
        return L == 16 ? CH_OK : CH_ERR_BODY;
    if (L < 20)                                 /* no room for count */
        return CH_SUCC_LEN;
    const int32_t c = (int32_t)be32_at(b + 20);
    h->count = c;
    if (c < -1)
        return CH_NEG_COUNT;
    if ((int64_t)L < 20 + 5 * (int64_t)(c > 0 ? c : 0))
        return CH_SUCC_LEN;
    return CH_OK;
}

/* children_head(), then the xid against xid_base + k.  Notifications and pings pass with their kind set. */
RG_HD uint32_t children_check(const uint8_t *b, uint64_t avail, int32_t xid_base, uint64_t d, uint64_t k, ChildHead *h)
{
    const uint32_t c = children_head(b, avail, xid_base, d, h);
    if (c != CH_OK || h->kind != RK_REPLY)
        return c;
    if ((uint32_t)h->xid != (uint32_t)xid_base + (uint32_t)k)
        return CH_ORDER;
    return CH_OK;
}

/* The listing entry at e, with `room` bytes to the end of its frame: a length word, L >= 1 name bytes that fit, and a
   name with no '/' and no NUL (the first such byte decides) that is not "." or "..".  *L = the name's length. */
RG_HD uint32_t children_entry(const uint8_t *e, uint64_t room, uint32_t *L)
{
    *L = 0;
    if (room < 4)
        return CH_ENT_TRUNC;
    const int32_t n = (int32_t)be32_at(e);
    if (n < 1)
        return CH_ENT_EMPTY;
    if ((uint64_t)n + 4u > room)
        return CH_ENT_TRUNC;
    *L = (uint32_t)n;
    for (uint32_t i = 0; i < (uint32_t)n; i++) {
        const uint8_t c = e[4 + i];
        if (c == '/')
            return CH_NAME_SLASH;
        if (c == 0)
            return CH_NAME_NUL;
    }
    if (e[4] == '.' && (n == 1 || (n == 2 && e[5] == '.')))
        return CH_NAME_DOT;
    return CH_OK;
}

}  /* namespace regk */

#if defined(__CUDACC__)
#include "regk_mkdirp.cuh"

namespace regk {

/* counters[]: RQ_ERR .. RQ_STOP as regk_replies.cuh uses them, then these */
enum { CQ_ENT_ERR = RQ_NCOUNTERS, CQ_NENT, CQ_MAXC, CQ_STALE, CQ_LISTED, CQ_UNLISTED, CQ_PREFIXES, CQ_NCOUNTERS };

struct ChParams {
    RepParams r;                                /* the frame chain (r.n = d) or the entry chain of one pass */
    uint64_t start;
    uint64_t d;                                 /* directories listed */
    uint64_t d_eff;                             /* replies the entry passes cover: those before the first frame fault */
    /* per directory k < d */
    unsigned long long *fpos;                   /* the reply frame's position */
    unsigned long long *fend;                   /* ... and its end */
    int32_t *err;
    uint32_t *cnt;                              /* max(count, 0) of a success, else 0 */
    uint32_t *seed_g;                           /* rank of the frame's first entry (RP_NONE: not a candidate) */
    uint32_t *last_g1;                          /* 1 + the largest rank of the frame's marked entries, 0 = none */
    uint32_t *name_bad;                         /* smallest rank of a marked entry whose name fails, RP_NONE = none */
    unsigned long long *end_pos;                /* where the frame's entry chain stops (q + 4 + L of its last entry) */
    unsigned long long *fault_pos;              /* position of the frame's entry fault */
    unsigned long long *child_off;              /* [d + 1] */
    const uint32_t *dir_len;                    /* [d] */
    /* the entry chain (in r: word, totals, tile_base, cand = entry candidates, marked) and the marked entries */
    const uint32_t *j0;                         /* successor of each entry candidate */
    unsigned long long *ent_pos;                /* [n_children] position of entry g's length word */
    uint32_t *ent_nlen;                         /* name length */
    uint32_t *ent_k;                            /* directory */
    uint32_t *ent_plen;                         /* listing path length: dir_len + 1 + L */
};

__device__ __forceinline__ uint32_t ch_cand_index(const RepParams &p, unsigned long long q)
{
    if (q >= p.len)
        return RP_NONE;
    const uint32_t w = p.word[q >> 4], f = (uint32_t)(q & 15u);
    if (!((w >> f) & 1u))
        return RP_NONE;
    return (uint32_t)(p.tile_base[q / RP_SPAN] + (w >> 16) + (uint32_t)__popc(w & ((1u << f) - 1u)));
}

/* the last frame k < m with fpos[k] <= q within [lo, hi], or lo - 1 (as a signed index) when none */
__device__ __forceinline__ long long ch_frame_of(const unsigned long long *fpos, long long lo, long long hi, unsigned long long q)
{
    long long a = lo - 1, b = hi;               /* fpos[a] <= q (virtually for lo - 1), answer in [a, b] */
    while (a < b) {
        const long long mid = (a + b + 1) >> 1;
        if (fpos[mid] <= q)
            a = mid;
        else
            b = mid - 1;
    }
    return a;
}

/* ---- frames, cand: the plausible frame positions at or after start ---- */
__global__ void __launch_bounds__(RP_TILE) regk_children_cand_kernel(const ChParams cp)
{
    const RepParams &p = cp.r;
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
    if (b < nblk && 16ull * b + 16u > cp.start) {
        for (uint32_t f = 0; f < 16u; f++) {
            const uint64_t pos = 16ull * b + f;
            if (pos >= p.len)
                break;
            ChildHead h;
            if (pos >= cp.start && children_head(s_win + 16u * threadIdx.x + f, p.len - pos, p.xid_base, p.n, &h) == CH_OK)
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

/* ---- seeds: mark the candidate at (pos[i] or 0) + add for every i < m whose cnt[i] (if given) is not 0 ---- */
__global__ void __launch_bounds__(256) regk_children_seed_kernel(const RepParams p, const unsigned long long *pos,
    const uint32_t *cnt, uint64_t m, unsigned long long add)
{
    const uint64_t i = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= m || (cnt && cnt[i] == 0u))
        return;
    const uint32_t c = ch_cand_index(p, (pos ? pos[i] : 0ull) + add);
    if (c != RP_NONE)
        p.marked[c] = 1;
}

/* ---- frames, chain: k of every reply frame, the check of k < d, the per-directory arrays ---- */
__global__ void __launch_bounds__(RP_TILE) regk_children_chain_kernel(const ChParams cp)
{
    const RepParams &p = cp.r;
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
            ChildHead h;
            const uint32_t code = children_check(p.s + pos, p.len - pos, p.xid_base, p.n, k, &h);
            cp.fpos[k] = pos;
            if (code != CH_OK) {
                atomicMin(p.counters + RQ_ERR, (unsigned long long)k << 8 | code);
            } else {
                const uint32_t n_ent = h.err == 0 && h.count > 0 ? (uint32_t)h.count : 0u;
                cp.err[k] = h.err;
                cp.cnt[k] = n_ent;
                cp.fend[k] = pos + 4u + (uint32_t)h.len;
                atomicAdd(&s_cnt[h.err == 0 ? 1 : h.err == -101 ? 2 : 3], 1u);
                if (n_ent)
                    atomicMax(p.counters + CQ_MAXC, (unsigned long long)n_ent);
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

/* ---- entries, cand: positions inside the bodies of frames k < d_eff with entries ---- */
__global__ void __launch_bounds__(RP_TILE) regk_children_ent_cand_kernel(const ChParams cp)
{
    const RepParams &p = cp.r;
    __shared__ __align__(16) uint8_t s_win[RP_SPAN + 32];
    __shared__ uint32_t s_warp[WARPS];
    __shared__ long long s_k[2];
    const uint64_t nblk = (p.len + 15u) / 16u;
    const uint64_t b0 = (uint64_t)blockIdx.x * RP_TILE, b = b0 + threadIdx.x;
    const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
    reinterpret_cast<uint4 *>(s_win)[threadIdx.x] = b < nblk ? rp_block(p.s, p.len, b) : zero;
    if (threadIdx.x < 2) {
        const uint64_t e = b0 + RP_TILE + threadIdx.x;
        reinterpret_cast<uint4 *>(s_win)[RP_TILE + threadIdx.x] = e < nblk ? rp_block(p.s, p.len, e) : zero;
        /* the frames this CTA's span can lie in: [frame of its first byte, frame of its last byte] */
        const unsigned long long q = threadIdx.x == 0 ? 16ull * b0 : 16ull * (b0 + RP_TILE) - 1u;
        s_k[threadIdx.x] = ch_frame_of(cp.fpos, 0, (long long)cp.d_eff - 1, q);
    }
    __syncthreads();
    uint32_t mask = 0;
    if (b < nblk && s_k[1] >= 0) {
        long long k = ch_frame_of(cp.fpos, s_k[0] < 0 ? 0 : s_k[0], s_k[1], 16ull * b);
        for (uint32_t f = 0; f < 16u; f++) {
            const uint64_t q = 16ull * b + f;
            if (q >= p.len)
                break;
            while (k + 1 < (long long)cp.d_eff && cp.fpos[k + 1] <= q)
                k++;
            if (k < 0 || cp.cnt[k] == 0u || q < cp.fpos[k] + 24u)
                continue;
            const unsigned long long E = cp.fend[k];
            if (q + 4u > E)
                continue;
            const uint8_t *e = s_win + 16u * threadIdx.x + f;
            const int32_t L = (int32_t)be32_at(e);
            if (L >= 1 && q + 4u + (uint32_t)L <= E && e[4] != 0 && e[4] != '/')
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

/* ---- entries: per-CTA counts of the marked entry candidates ---- */
__global__ void __launch_bounds__(RP_TILE) regk_children_ent_count_kernel(const RepParams p)
{
    const uint64_t c = (uint64_t)blockIdx.x * RP_TILE + threadIdx.x;
    const uint32_t cnt = (uint32_t)__popc(__ballot_sync(0xFFFFFFFFu, c < p.C && p.marked[c]));
    if ((threadIdx.x & 31u) == 0)
        add_tile_total(p.tile_total, p.super_total, blockIdx.x, cnt);
}

/* ---- entries: rank g of every marked entry, its directory, its name check, where its frame's chain stops ---- */
__global__ void __launch_bounds__(RP_TILE) regk_children_ent_kernel(const ChParams cp)
{
    const RepParams &p = cp.r;
    __shared__ uint32_t s_warp[WARPS];
    __shared__ unsigned long long s_base;
    if (threadIdx.x < 32) {
        const unsigned long long base = tile_base_from_totals(p.tile_total, p.super_total, blockIdx.x);
        if (threadIdx.x == 0)
            s_base = base;
    }
    const uint64_t c = (uint64_t)blockIdx.x * RP_TILE + threadIdx.x;
    const bool on = c < p.C && p.marked[c];
    uint32_t tot;
    const uint32_t r = block_scan<uint32_t>(s_warp, on ? 1u : 0u, &tot);
    if (on) {
        const uint32_t g = (uint32_t)(s_base + r);
        const unsigned long long q = p.cand[c];
        const uint32_t k = (uint32_t)ch_frame_of(cp.fpos, 0, (long long)cp.d_eff - 1, q);
        uint32_t L;
        const uint32_t code = children_entry(p.s + q, cp.fend[k] - q, &L);
        cp.ent_pos[g] = q;
        cp.ent_nlen[g] = L;
        cp.ent_k[g] = k;
        cp.ent_plen[g] = cp.dir_len[k] + 1u + L;
        if (q == cp.fpos[k] + 24u)
            cp.seed_g[k] = g;
        if (code != CH_OK)
            atomicMin(cp.name_bad + k, g);
        atomicMax(cp.last_g1 + k, g + 1u);
        if (cp.j0[c] == RP_NONE)
            cp.end_pos[k] = q + 4u + L;
    }
    if (c + 1 == p.C)
        p.counters[CQ_NENT] = s_base + tot;
}

/* ---- entries, per frame: the chain against the count (the first fault a front-to-back reader meets), child_off ---- */
__global__ void __launch_bounds__(256) regk_children_ent_frame_kernel(const ChParams cp)
{
    const RepParams &p = cp.r;
    const uint64_t k = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (k >= cp.d_eff)
        return;
    const unsigned long long F = cp.fpos[k], E = cp.fend[k];
    const uint64_t ne = p.counters[CQ_NENT];
    {
        uint64_t a = 0, b = ne;                     /* lower bound of F in ent_pos: the entries of earlier frames */
        while (a < b) {
            const uint64_t mid = (a + b) >> 1;
            if (cp.ent_pos[mid] < F)
                a = mid + 1;
            else
                b = mid;
        }
        cp.child_off[k] = a;
    }
    if (cp.err[k] != 0)
        return;
    const uint32_t c = cp.cnt[k];
    unsigned long long pos = ~0ull;
    uint32_t code = CH_OK;
    if (c == 0u) {
        if (E != F + 24u) {
            pos = F + 24u;
            code = CH_ENT_END;
        }
    } else {
        const uint32_t sg = cp.seed_g[k];
        const uint32_t m = sg == RP_NONE ? 0u : cp.last_g1[k] - sg;
        const uint32_t nb = cp.name_bad[k];
        const uint32_t i_name = nb == RP_NONE ? RP_NONE : nb - sg;
        const uint32_t fi = min(i_name, m < c ? m : RP_NONE);
        if (fi < c) {
            pos = fi == i_name ? cp.ent_pos[nb] : (m == 0u ? F + 24u : cp.end_pos[k]);
            uint32_t L;
            code = children_entry(p.s + pos, E - pos, &L);
        } else if (c < m) {
            pos = cp.ent_pos[sg + c];
            code = CH_ENT_END;
        } else if (cp.end_pos[k] != E) {
            pos = cp.end_pos[k];
            code = CH_ENT_END;
        }
    }
    if (code != CH_OK) {
        cp.fault_pos[k] = pos;
        atomicMin(p.counters + CQ_ENT_ERR, (unsigned long long)k << 8 | code);
    }
}

/* ---- listing: path e = directory + '/' + name, output-stationary 16-byte blocks (as regk_mkdirp_gather_kernel) ---- */
struct ChGatherParams {
    uint64_t n;                                 /* listing entries */
    const unsigned long long *tile_total;       /* regk_mkdirp_len_kernel's totals of ent_plen */
    const unsigned long long *super_total;
    const uint32_t *ent_k, *ent_nlen, *ent_plen;
    const unsigned long long *ent_pos;
    const uint8_t *dir_bytes;                   /* the packed listed directories */
    const unsigned long long *dir_off;
    const uint8_t *s;                           /* the reply stream */
    uint8_t *out_bytes;
    unsigned long long *out_off;                /* [n + 1] */
};

__global__ void __launch_bounds__(MK_TILE) regk_children_gather_kernel(const ChGatherParams p)
{
    __shared__ unsigned long long s_warp[MK_TILE / 32];
    __shared__ unsigned long long s_off[MK_TILE + 1];
    __shared__ unsigned long long s_dir[MK_TILE];               /* where each entry's directory starts */
    __shared__ unsigned long long s_name[MK_TILE];              /* where its name starts in the stream */
    __shared__ uint32_t s_dlen[MK_TILE];
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
    const uint64_t g0 = (uint64_t)tile * MK_TILE, g = g0 + threadIdx.x;
    const uint32_t ng = (uint32_t)min((uint64_t)MK_TILE, p.n - g0);
    const unsigned long long len = threadIdx.x < ng ? p.ent_plen[g] : 0ull;
    if (threadIdx.x < ng) {
        const uint32_t k = p.ent_k[g];
        s_dir[threadIdx.x] = p.dir_off[k];
        s_dlen[threadIdx.x] = (uint32_t)(p.dir_off[k + 1] - p.dir_off[k]);
        s_name[threadIdx.x] = p.ent_pos[g] + 4u;
    }
    unsigned long long total;
    const unsigned long long excl = block_scan<unsigned long long>(s_warp, len, &total);
    const unsigned long long base = s_base;
    if (threadIdx.x < ng) {
        s_off[threadIdx.x] = excl;
        p.out_off[g] = base + excl;
    }
    if (threadIdx.x == 0)
        s_off[ng] = total;
    if (g0 + ng == p.n && threadIdx.x == 0)
        p.out_off[p.n] = base + total;
    __syncthreads();
    const unsigned long long a0 = base & ~15ull;
    const uint32_t lead = (uint32_t)(base - a0);
    const unsigned long long nblk = (lead + total + 15ull) >> 4;
    for (unsigned long long b = threadIdx.x; b < nblk; b += MK_TILE) {
        const long long bs = (long long)(16ull * b) - (long long)lead;
        const unsigned long long pos0 = bs < 0 ? 0ull : (unsigned long long)bs;
        const unsigned long long end = min((unsigned long long)(bs + 16), total);
        uint32_t lo = 0, hi = ng - 1u;
        while (lo < hi) {
            const uint32_t mid = (lo + hi + 1u) >> 1;
            if (s_off[mid] <= pos0)
                lo = mid;
            else
                hi = mid - 1u;
        }
        uint32_t e = lo;
        uint32_t acc[4] = {0u, 0u, 0u, 0u};
        for (unsigned long long q = pos0; q < end; q++) {
            while (q >= s_off[e + 1])
                e++;
            const unsigned long long t = q - s_off[e];
            const uint32_t dl = s_dlen[e];
            const uint32_t byte = t < dl ? p.dir_bytes[s_dir[e] + t] : t == dl ? (uint32_t)'/' : p.s[s_name[e] + (t - dl - 1u)];
            const uint32_t lanebyte = (uint32_t)(q - (unsigned long long)bs);
            acc[lanebyte >> 2] |= byte << (8u * (lanebyte & 3u));
        }
        uint8_t *gp = p.out_bytes + a0 + 16ull * b;
        if (bs >= 0 && (unsigned long long)bs + 16ull <= total) {
            stg_v4(gp, make_uint4(acc[0], acc[1], acc[2], acc[3]));
        } else {
            for (unsigned long long q = pos0; q < end; q++) {
                const uint32_t lanebyte = (uint32_t)(q - (unsigned long long)bs);
                gp[lanebyte] = (uint8_t)(acc[lanebyte >> 2] >> (8u * (lanebyte & 3u)));
            }
        }
    }
}

/* ---- the directory set: the distinct parents of the batch, listed (valid, not "/") or not, in parent order ---- */
struct ChDirParams {
    const uint8_t *path_bytes;
    const unsigned long long *path_off;
    const uint32_t *parent_len;
    const unsigned long long *unique_first;
    uint64_t nu;
    uint32_t *tile_a, *tile_b;                  /* unlisted / listed counts, two-level */
    unsigned long long *super_a, *super_b;
    unsigned long long *counters;
    unsigned long long *unlisted;               /* first records of "/" and rejected directories */
    unsigned long long *dir_rec;                /* listed: first record, length */
    uint32_t *dir_len;
};

__device__ __forceinline__ uint32_t ch_dir_class(const ChDirParams &p, uint64_t u, uint32_t *depth)
{
    const uint64_t r = p.unique_first[u];
    const uint32_t c = mkdir_components(p.path_bytes + p.path_off[r], p.parent_len[r]);
    *depth = c == MKDIR_INVALID ? 0u : c;
    return c == MKDIR_INVALID || c == 0u ? 1u : 2u;     /* 1 unlisted, 2 listed */
}

__global__ void __launch_bounds__(MK_TILE) regk_children_dirs_count_kernel(const ChDirParams p)
{
    const uint64_t u = (uint64_t)blockIdx.x * MK_TILE + threadIdx.x;
    uint32_t f = 0, depth = 0;
    if (u < p.nu)
        f = ch_dir_class(p, u, &depth);
    const uint32_t na = __popc(__ballot_sync(0xFFFFFFFFu, f == 1u)), nb = __popc(__ballot_sync(0xFFFFFFFFu, f == 2u));
    unsigned long long e = depth;
    #pragma unroll
    for (int d = 16; d > 0; d >>= 1)
        e += __shfl_xor_sync(0xFFFFFFFFu, e, d);
    if ((threadIdx.x & 31u) == 0) {
        add_tile_total(p.tile_a, p.super_a, blockIdx.x, na);
        add_tile_total(p.tile_b, p.super_b, blockIdx.x, nb);
        if (e)
            atomicAdd(p.counters + CQ_PREFIXES, e);     /* component-boundary prefixes of the listed ones */
    }
}

__global__ void __launch_bounds__(MK_TILE) regk_children_dirs_kernel(const ChDirParams p)
{
    __shared__ uint32_t s_warp[2][MK_TILE / 32];
    __shared__ unsigned long long s_base[2];
    const uint32_t tile = blockIdx.x, lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    if (threadIdx.x < 32) {
        const unsigned long long a = tile_base_from_totals(p.tile_a, p.super_a, tile);
        const unsigned long long b = tile_base_from_totals(p.tile_b, p.super_b, tile);
        if (threadIdx.x == 0) {
            s_base[0] = a;
            s_base[1] = b;
        }
    }
    const uint64_t u = (uint64_t)tile * MK_TILE + threadIdx.x;
    uint32_t f = 0, depth;
    if (u < p.nu)
        f = ch_dir_class(p, u, &depth);
    const uint32_t ba = __ballot_sync(0xFFFFFFFFu, f == 1u), bb = __ballot_sync(0xFFFFFFFFu, f == 2u);
    if (lane == 0) {
        s_warp[0][warp] = __popc(ba);
        s_warp[1][warp] = __popc(bb);
    }
    __syncthreads();
    uint32_t ra = __popc(ba & ((1u << lane) - 1u)), rb = __popc(bb & ((1u << lane) - 1u)), ta = 0, tb = 0;
    #pragma unroll
    for (uint32_t w = 0; w < MK_TILE / 32; w++) {
        if (w < warp) {
            ra += s_warp[0][w];
            rb += s_warp[1][w];
        }
        ta += s_warp[0][w];
        tb += s_warp[1][w];
    }
    if (f) {
        const unsigned long long r = p.unique_first[u];
        if (f == 1u) {
            p.unlisted[s_base[0] + ra] = r;
        } else {
            p.dir_rec[s_base[1] + rb] = r;
            p.dir_len[s_base[1] + rb] = p.parent_len[r];
        }
    }
    if (u + 1 == p.nu) {
        p.counters[CQ_UNLISTED] = s_base[0] + ta;
        p.counters[CQ_LISTED] = s_base[1] + tb;
    }
}

/* ---- keep: the batch's paths and the listed directories' prefixes in one table; listing paths probe it ---- */
struct ChKeepParams {
    const uint8_t *path_bytes;                  /* the batch's path stream (>= 16 bytes of slack) */
    const unsigned long long *path_off;
    uint64_t n;
    const unsigned long long *dir_rec;          /* listed directories */
    const uint32_t *dir_len;
    uint64_t d;
    unsigned long long *table;                  /* (record + 1) << 32 | length, 0 = empty (zeroed by the host) */
    uint32_t mask;
    /* the listing and its classes */
    const uint8_t *lst_bytes;                   /* (>= 16 bytes of slack) */
    const unsigned long long *lst_off;
    uint64_t n_children;
    uint8_t *cls;
    uint32_t *tile_total;
    unsigned long long *super_total;
    unsigned long long *stale;
    uint32_t *stale_len;
    unsigned long long *counters;
};

__device__ __forceinline__ void ch_keep_insert(const ChKeepParams &p, uint32_t r, uint32_t L)
{
    const uint32_t *W = reinterpret_cast<const uint32_t *>(p.path_bytes);
    const unsigned long long o = p.path_off[r];
    const unsigned long long key = ((unsigned long long)(r + 1u) << 32) | L;
    uint32_t slot = string_hash32(W, o, L) & p.mask;
    for (;;) {
        unsigned long long cur = p.table[slot];
        if (cur == 0ull) {
            cur = atomicCAS(p.table + slot, 0ull, key);
            if (cur == 0ull)
                return;
        }
        if ((uint32_t)cur == L) {
            const uint32_t j = (uint32_t)(cur >> 32) - 1u;
            if (j == r || string_equal(W, o, p.path_off[j], L))
                return;
        }
        slot = (slot + 1u) & p.mask;
    }
}

__global__ void __launch_bounds__(256) regk_children_keep_paths_kernel(const ChKeepParams p)
{
    const uint64_t i = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (i < p.n)
        ch_keep_insert(p, (uint32_t)i, (uint32_t)(p.path_off[i + 1] - p.path_off[i]));
}

/* one thread per listed directory: each prefix that ends before a '/' of it, and the directory itself */
__global__ void __launch_bounds__(256) regk_children_keep_dirs_kernel(const ChKeepParams p)
{
    const uint64_t j = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (j >= p.d)
        return;
    const uint32_t r = (uint32_t)p.dir_rec[j], L = p.dir_len[j];
    const uint8_t *b = p.path_bytes + p.path_off[r];
    for (uint32_t t = 1; t < L; t++)
        if (b[t] == '/')
            ch_keep_insert(p, r, t);
    ch_keep_insert(p, r, L);
}

__global__ void __launch_bounds__(MK_TILE) regk_children_probe_kernel(const ChKeepParams p)
{
    const uint64_t g = (uint64_t)blockIdx.x * MK_TILE + threadIdx.x;
    bool stale = false;
    if (g < p.n_children) {
        const uint32_t *W = reinterpret_cast<const uint32_t *>(p.path_bytes);
        const uint32_t *V = reinterpret_cast<const uint32_t *>(p.lst_bytes);
        const unsigned long long o = p.lst_off[g];
        const uint32_t L = (uint32_t)(p.lst_off[g + 1] - o);
        uint32_t slot = string_hash32(V, o, L) & p.mask;
        stale = true;
        for (;;) {
            const unsigned long long cur = p.table[slot];
            if (cur == 0ull)
                break;
            if ((uint32_t)cur == L &&
                string_equal2(W, p.path_off[(uint32_t)(cur >> 32) - 1u], ~0ull, V, o, ~0ull, L)) {
                stale = false;
                break;
            }
            slot = (slot + 1u) & p.mask;
        }
        p.cls[g] = stale ? 1u : 0u;
    }
    const uint32_t cnt = (uint32_t)__popc(__ballot_sync(0xFFFFFFFFu, stale));
    if ((threadIdx.x & 31u) == 0)
        add_tile_total(p.tile_total, p.super_total, blockIdx.x, cnt);
}

__global__ void __launch_bounds__(MK_TILE) regk_children_stale_kernel(const ChKeepParams p)
{
    __shared__ uint32_t s_warp[WARPS];
    __shared__ unsigned long long s_base;
    if (threadIdx.x < 32) {
        const unsigned long long base = tile_base_from_totals(p.tile_total, p.super_total, blockIdx.x);
        if (threadIdx.x == 0)
            s_base = base;
    }
    const uint64_t g = (uint64_t)blockIdx.x * MK_TILE + threadIdx.x;
    const bool st = g < p.n_children && p.cls[g] != 0;
    uint32_t tot;
    const uint32_t r = block_scan<uint32_t>(s_warp, st ? 1u : 0u, &tot);
    if (st) {
        p.stale[s_base + r] = g;
        p.stale_len[s_base + r] = (uint32_t)(p.lst_off[g + 1] - p.lst_off[g]);
    }
    if (g + 1 == p.n_children)
        p.counters[CQ_STALE] = s_base + tot;
}

}  /* namespace regk */
#endif /* __CUDACC__ */
#endif /* REGK_CHILDREN_CUH */
