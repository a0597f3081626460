/*
 * regk_walk.cuh — walk a registry subtree level by level: getData and getChildren for every node of the frontier,
 * the found nodes appended to one breadth-first snapshot, the listed children the next frontier.  The batch form of
 * Binder's own access pattern (fetch a node, list its children, fetch every child), one round trip per tree level.
 *
 * The frontier of f nodes is a packed path stream that starts at 0 (the roots, or the listing paths of the previous
 * level), so node i's frames start at closed-form offsets:
 *   frame i      (getData)     at 17 i + path_off[i]
 *   frame f + i  (getChildren) at S + 17 i + path_off[i],  S = 17 f + path_off[f] (the getData section's size)
 * The reply sections are read by the existing passes, launched from the walk's host driver on buffers of its own:
 *   getData      regk_replies.cuh's cand / compact / succ / jump / mark / chain_count / chain: err, data position,
 *                data length, Stat.version and Stat.ephemeralOwner per frontier node
 *   getChildren  regk_children.cuh's frame and entry passes from the getData section's end, and its listing gather
 *                (directory + '/' + name, from the frontier's packed paths): the next frontier
 *   packing      regk_mkdirp_len_kernel / regk_mkdirp_gather_kernel: the level's node paths (from the frontier) and
 *                data (from the reply stream), as regk_read_replies packs its snapshot
 * The passes here:
 *   frame        output-stationary: each CTA owns the bytes of 128 frames of one section and writes them as whole
 *                16-byte blocks (byte stores only at its ragged ends), with frame_off.
 *   found        the frontier nodes whose getData reply has err 0, compacted in frontier order with their stats and
 *                lengths (two-level totals, block scan); per-CTA counts of err 0 / NONODE / other.
 *   append       one level's packed stream appended to the walk's snapshot stream at its current end: offsets shifted,
 *                bytes written as whole 16-byte blocks of the destination.  The host grows the snapshot geometrically,
 *                so earlier levels are copied O(log levels) times in all, not once per level.
 */
#ifndef REGK_WALK_CUH
#define REGK_WALK_CUH

#include "regk_children.cuh"

namespace regk {

/* ---- frame: getData then getChildren frames of the frontier ---- */
struct WalkFrameParams {
    uint64_t f;                                 /* frontier nodes */
    const uint8_t *path_bytes;                  /* the frontier's packed paths */
    const unsigned long long *path_off;         /* [f + 1], path_off[0] == 0 */
    int32_t xid_base;
    unsigned long long sec1;                    /* 17 f + path_off[f]: where the getChildren section starts */
    uint8_t *out;                               /* [2 sec1], 16-byte aligned */
    unsigned long long *out_off;                /* [2 f + 1] */
};

__device__ __forceinline__ uint32_t wk_be_byte(uint32_t v, uint32_t k)
{
    return (v >> (8u * (3u - k))) & 0xFFu;
}

__global__ void __launch_bounds__(MK_TILE) regk_walk_frame_kernel(const WalkFrameParams p)
{
    __shared__ unsigned long long s_off[MK_TILE + 1];           /* tile-relative frame starts */
    __shared__ unsigned long long s_src[MK_TILE];               /* where each frame's path starts in the path stream */
    const uint64_t tiles = (p.f + MK_TILE - 1) / MK_TILE;
    const uint32_t sec = (uint64_t)blockIdx.x >= tiles ? 1u : 0u;
    const uint64_t i0 = ((uint64_t)blockIdx.x - sec * tiles) * MK_TILE;
    const uint32_t ni = (uint32_t)min((uint64_t)MK_TILE, p.f - i0);
    const unsigned long long sbase = sec ? p.sec1 : 0ull, p0 = p.path_off[i0];
    const unsigned long long base = sbase + 17ull * i0 + p0;
    if (threadIdx.x < ni) {
        const uint64_t k = i0 + threadIdx.x;
        const unsigned long long pk = p.path_off[k];
        s_off[threadIdx.x] = 17ull * threadIdx.x + pk - p0;
        s_src[threadIdx.x] = pk;
        p.out_off[sec * p.f + k] = sbase + 17ull * k + pk;
    }
    if (threadIdx.x == 0) {
        s_off[ni] = 17ull * ni + p.path_off[i0 + ni] - p0;
        if (sec == 1u && i0 + ni == p.f)
            p.out_off[2 * p.f] = 2 * p.sec1;
    }
    __syncthreads();
    const unsigned long long total = s_off[ni];
    const uint32_t op = sec ? 8u : 4u;
    const uint32_t xb = (uint32_t)p.xid_base + (sec ? (uint32_t)p.f : 0u) + (uint32_t)i0;
    const unsigned long long a0 = base & ~15ull;
    const uint32_t lead = (uint32_t)(base - a0);
    const unsigned long long nblk = (lead + total + 15ull) >> 4;
    for (unsigned long long b = threadIdx.x; b < nblk; b += MK_TILE) {
        const long long bs = (long long)(16ull * b) - (long long)lead;   /* tile-relative byte of the block's lane 0 */
        const unsigned long long pos0 = bs < 0 ? 0ull : (unsigned long long)bs;
        const unsigned long long end = min((unsigned long long)(bs + 16), total);
        uint32_t lo = 0, hi = ni - 1u;                          /* the frame pos0 lies in: last s_off[e] <= pos0 */
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
            const uint32_t t = (uint32_t)(q - s_off[e]);
            const uint32_t P = (uint32_t)(s_off[e + 1] - s_off[e]) - 17u;
            uint32_t byte;
            if (t < 4u)
                byte = wk_be_byte(13u + P, t);
            else if (t < 8u)
                byte = wk_be_byte(xb + e, t - 4u);
            else if (t < 12u)
                byte = wk_be_byte(op, t - 8u);
            else if (t < 16u)
                byte = wk_be_byte(P, t - 12u);
            else if (t < 16u + P)
                byte = p.path_bytes[s_src[e] + (t - 16u)];
            else
                byte = 0u;                                      /* watch = false */
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

/* ---- found: the frontier nodes whose getData reply has err 0, in frontier order ---- */
enum { WK_FOUND = 0, WK_MISSING, WK_ERROR, WK_NCOUNTERS };

struct WalkFoundParams {
    uint64_t f;
    const int32_t *err;                         /* per frontier node, from the getData chain */
    const uint32_t *dlen;
    const int32_t *ver;
    const long long *own;
    const unsigned long long *path_off;         /* the frontier's [f + 1] */
    uint32_t *tile_total;
    unsigned long long *super_total;
    unsigned long long *node_rec;               /* [found] frontier node */
    int32_t *node_ver;
    long long *node_own;
    uint32_t *node_plen, *node_dlen;
    unsigned long long *counters;               /* [WK_NCOUNTERS] */
};

__global__ void __launch_bounds__(RP_TILE) regk_walk_found_count_kernel(const WalkFoundParams p)
{
    __shared__ uint32_t s_cnt[3];
    if (threadIdx.x < 3)
        s_cnt[threadIdx.x] = 0;
    __syncthreads();
    const uint64_t i = (uint64_t)blockIdx.x * RP_TILE + threadIdx.x;
    const int32_t e = i < p.f ? p.err[i] : 1;
    const uint32_t cnt = (uint32_t)__popc(__ballot_sync(0xFFFFFFFFu, e == 0));
    if ((threadIdx.x & 31u) == 0)
        add_tile_total(p.tile_total, p.super_total, blockIdx.x, cnt);
    if (i < p.f)
        atomicAdd(&s_cnt[e == 0 ? 0 : e == -101 ? 1 : 2], 1u);
    __syncthreads();
    if (threadIdx.x < 3 && s_cnt[threadIdx.x])
        atomicAdd(p.counters + WK_FOUND + threadIdx.x, (unsigned long long)s_cnt[threadIdx.x]);
}

__global__ void __launch_bounds__(RP_TILE) regk_walk_found_kernel(const WalkFoundParams p)
{
    __shared__ uint32_t s_warp[WARPS];
    __shared__ unsigned long long s_base;
    if (threadIdx.x < 32) {
        const unsigned long long base = tile_base_from_totals(p.tile_total, p.super_total, blockIdx.x);
        if (threadIdx.x == 0)
            s_base = base;
    }
    const uint64_t i = (uint64_t)blockIdx.x * RP_TILE + threadIdx.x;
    const bool found = i < p.f && p.err[i] == 0;
    uint32_t tot;
    const uint32_t r = block_scan<uint32_t>(s_warp, found ? 1u : 0u, &tot);   /* its barriers publish s_base */
    if (found) {
        const uint64_t j = s_base + r;
        p.node_rec[j] = i;
        p.node_ver[j] = p.ver[i];
        p.node_own[j] = p.own[i];
        p.node_plen[j] = (uint32_t)(p.path_off[i + 1] - p.path_off[i]);
        p.node_dlen[j] = p.dlen[i];
    }
}

/* ---- append: a level's packed stream and offsets at the end of the snapshot's ---- */
struct WalkAppendParams {
    const uint8_t *src;                         /* the level's bytes, [0, len) */
    unsigned long long len;
    uint8_t *dst;                               /* the snapshot stream (16-byte aligned); the level goes to [at, at + len) */
    unsigned long long at;
    const unsigned long long *src_off;          /* [n + 1], from 0 */
    uint64_t n;
    unsigned long long *dst_off;                /* the snapshot's offsets from the level's first node: [n + 1] */
};

__global__ void __launch_bounds__(256) regk_walk_append_kernel(const WalkAppendParams p)
{
    const uint64_t t = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (t <= p.n)
        p.dst_off[t] = p.at + p.src_off[t];
    const unsigned long long a0 = p.at & ~15ull, lo = p.at, hi = p.at + p.len;
    const unsigned long long q0 = a0 + 16ull * t;
    if (q0 >= hi)
        return;
    uint32_t acc[4] = {0u, 0u, 0u, 0u};
    #pragma unroll
    for (uint32_t k = 0; k < 16u; k++) {
        const unsigned long long q = q0 + k;
        if (q >= lo && q < hi)
            acc[k >> 2] |= (uint32_t)p.src[q - lo] << (8u * (k & 3u));
    }
    if (q0 >= lo && q0 + 16u <= hi) {
        stg_v4(p.dst + q0, make_uint4(acc[0], acc[1], acc[2], acc[3]));
    } else {                                    /* the first and last block: the level's own bytes only */
        for (uint32_t k = 0; k < 16u; k++) {
            const unsigned long long q = q0 + k;
            if (q >= lo && q < hi)
                p.dst[q] = (uint8_t)(acc[k >> 2] >> (8u * (k & 3u)));
        }
    }
}

}  /* namespace regk */
#endif /* REGK_WALK_CUH */
