/*
 * regk_walk_setwatches.cuh — carry a watched walk across a reconnect: the watches each snapshot node holds, and the
 * SetWatches frames (op 101) for them (regk_walk_setwatches).
 *
 * armed     one byte per snapshot node: 1 when the last read of the node was framed with REGK_ZK_WATCH and both its
 *           getData and its getChildren reply had err 0, so the session holds its data and its child watch.
 *             arm         after a watched read: a plain level's found node k (appended as node base + k) from its
 *                         frontier node's getChildren err; a refresh level's frontier node i (snapshot node fnode[i])
 *                         from both errs.  An unwatched read, or any err, clears the byte.
 *             keep armed  the bytes compacted alongside regk_walk_keep_kernel, from its own tile totals and predicate
 *                         (the nodes not marked removed), so the byte moves with its node through a rebuild.
 * framing   classify (one thread per snapshot node: LISTED when armed and neither pending, removed nor a node of the
 *           refresh frontier; REPEND when it is none of those either; per-tile count and bytes 4 + P of the listed
 *           nodes), then place (the tile look-back of those totals: listed node j's D entry at index r_j and prefix s_j,
 *           its C entry at nD + r_j and bD + s_j; a REPEND node marked pending).  Place runs only after every buffer
 *           the call needs is reserved, so a failed allocation leaves no node re-pended.  regk_setwatches.cuh's lmax,
 *           write and head kernels finish the frames, with nE = 0.
 */
#ifndef REGK_WALK_SETWATCHES_CUH
#define REGK_WALK_SETWATCHES_CUH

#include "regk_setwatches.cuh"
#include "regk_walk_watch.cuh"

namespace regk {

enum : uint8_t { WS_NONE = 0, WS_LISTED = 1, WS_REPEND = 2 };

/* ---- arm: the armed byte of the nodes a watched (or unwatched) read just read ---- */
struct WalkArmParams {
    uint64_t n;                                 /* found nodes (plain level) or frontier nodes (refresh level) */
    const unsigned long long *node_rec;         /* plain: [n] the frontier node of found node k; NULL on a refresh level */
    const unsigned long long *fnode;            /* refresh: [n] the snapshot node of frontier node i */
    uint64_t base;                              /* plain: found node k is snapshot node base + k */
    const int32_t *err, *cerr;                  /* per frontier node: getData err, getChildren err */
    uint32_t watch;
    uint8_t *armed;
};

__global__ void __launch_bounds__(256) regk_walk_arm_kernel(const WalkArmParams p)
{
    const uint64_t k = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (k >= p.n)
        return;
    const uint64_t i = p.node_rec ? p.node_rec[k] : k;
    const uint64_t j = p.node_rec ? p.base + k : p.fnode[k];
    const bool ok = p.watch && p.err[i] == 0 && p.cerr[i] == 0;
    p.armed[j] = ok ? 1u : 0u;
}

/* ---- keep armed: regk_walk_keep_kernel's compaction of the armed bytes (its tile totals, its predicate) ---- */
__global__ void __launch_bounds__(RP_TILE) regk_walk_keep_armed_kernel(const WalkKeepParams p, const uint8_t *armed,
    uint8_t *narmed)
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
    if (keep)
        narmed[s_base + r] = armed[j];
}

/* ---- classify / place over the snapshot's m nodes ---- */
struct WalkSwParams {
    uint64_t m;
    const unsigned long long *path_off;         /* the snapshot's [m + 1] */
    const uint8_t *armed;
    uint32_t *mark;
    const unsigned long long *fnode;            /* the refresh frontier, ascending; f = 0 when there is none */
    uint64_t f;
    uint8_t *cls;                               /* [m] WS_* */
    uint32_t *tt[2];                            /* tile totals: listed count, listed bytes */
    unsigned long long *st[2];
    unsigned long long *counters;               /* [1] re-pended */
    /* place */
    uint64_t nD, bD;
    unsigned long long *ent_src, *ent_s;        /* [2 nD] */
    uint32_t *ent_len;
};

/* node j is a node of the refresh frontier (fnode is ascending) */
__device__ __forceinline__ bool ws_in_frontier(const WalkSwParams &p, uint64_t j)
{
    uint64_t lo = 0, hi = p.f;
    while (lo < hi) {
        const uint64_t mid = (lo + hi) >> 1;
        if (p.fnode[mid] < j)
            lo = mid + 1;
        else
            hi = mid;
    }
    return lo < p.f && p.fnode[lo] == j;
}

__global__ void __launch_bounds__(RP_TILE) regk_walk_sw_classify_kernel(const WalkSwParams p)
{
    const uint64_t j = (uint64_t)blockIdx.x * RP_TILE + threadIdx.x;
    uint32_t size = 0;
    uint8_t c = WS_NONE;
    if (j < p.m) {
        if (!(p.mark[j] & (WK_PENDING | WK_REMOVED)) && !ws_in_frontier(p, j))
            c = p.armed[j] ? WS_LISTED : WS_REPEND;
        if (c == WS_LISTED)
            size = 4u + (uint32_t)(p.path_off[j + 1] - p.path_off[j]);
        p.cls[j] = c;
    }
    const uint32_t cnt = __popc(__ballot_sync(0xFFFFFFFFu, c == WS_LISTED));
    const uint32_t nrep = __popc(__ballot_sync(0xFFFFFFFFu, c == WS_REPEND));
    const uint32_t bytes = __reduce_add_sync(0xFFFFFFFFu, size);
    if ((threadIdx.x & 31u) == 0) {
        add_tile_total(p.tt[0], p.st[0], blockIdx.x, cnt);
        add_tile_total(p.tt[1], p.st[1], blockIdx.x, bytes);
        if (nrep)
            atomicAdd(p.counters, (unsigned long long)nrep);
    }
}

__global__ void __launch_bounds__(RP_TILE) regk_walk_sw_place_kernel(const WalkSwParams p)
{
    __shared__ unsigned long long s_warp[WARPS];
    __shared__ unsigned long long s_base[2];
    if (threadIdx.x < 32) {
        for (int q = 0; q < 2; q++) {
            const unsigned long long v = tile_base_from_totals(p.tt[q], p.st[q], blockIdx.x);
            if (threadIdx.x == 0)
                s_base[q] = v;
        }
    }
    const uint64_t j = (uint64_t)blockIdx.x * RP_TILE + threadIdx.x;
    const uint8_t c = j < p.m ? p.cls[j] : WS_NONE;
    const uint32_t P = c == WS_LISTED ? (uint32_t)(p.path_off[j + 1] - p.path_off[j]) : 0u;
    /* one scan of count << 40 | bytes; a CTA's bytes stay below 2^40 */
    const unsigned long long v = c == WS_LISTED ? (1ull << 40) | (4ull + P) : 0ull;
    unsigned long long tot;
    const unsigned long long x = block_scan<unsigned long long>(s_warp, v, &tot);     /* its barriers publish s_base */
    if (c == WS_REPEND) {
        p.mark[j] |= WK_PENDING;
    } else if (c == WS_LISTED) {
        const uint64_t r = s_base[0] + (x >> 40), s = s_base[1] + (x & ((1ull << 40) - 1));
        const unsigned long long src = p.path_off[j];
        p.ent_src[r] = src;
        p.ent_len[r] = P;
        p.ent_s[r] = s;
        p.ent_src[p.nD + r] = src;
        p.ent_len[p.nD + r] = P;
        p.ent_s[p.nD + r] = p.bD + s;
    }
}

}  /* namespace regk */
#endif /* REGK_WALK_SETWATCHES_CUH */
