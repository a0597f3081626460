/*
 * regk_reconcile.cuh — compare the batch finished last ("desired": n records, path i and payload i) with a snapshot
 * of the registry ("observed": m nodes, path j and data j) and list what repairs the difference.  Nodes are keyed by
 * their path bytes, compared byte for byte; a hash only picks a table slot.
 *
 *   cls[i]      DUP     an earlier record has the same path (the first occurrence decides, as ZooKeeper keeps the
 *                       first create)
 *               CREATE  no node has path i          UPDATE  the node's data differs from payload i
 *               SAME    the node holds payload i byte for byte
 *               REPLACE (stats present: regk_reconcile_owned) the node's ephemeral owner is not the one wanted; the
 *                       payload is not compared
 *   match[i]    the node with path i, or ~0 (DUP records carry their path's match too)
 *   obs_cls[j]  KEEP if some record has path j, else DELETE
 *
 * The passes, one kernel each (the host reads the counters once, after compaction):
 *   insert    one thread per node: a device snapshot's offsets are checked first (a bad node is reported as the
 *             smallest bad index and never read); then j + 1 goes into T_o, an open-addressing table of 32-bit slots,
 *             with the protocol of regk_parent_kernel: atomicCAS claims an empty slot, a slot whose node has the same
 *             path keeps the smaller index by atomicMin, any other slot moves on.
 *   desired   one thread per record: probe T_o read-only (match; with stats, the matched node's owner; then the
 *             payload comparison), then insert i + 1 into T_d with the same protocol.
 *   mark      records: DUP iff the T_d slot names another record.  Nodes: a node whose T_o slot names another node
 *             is a duplicate path (the call is refused, naming the smallest such index); the others probe T_d for
 *             KEEP / DELETE.  Per-tile counts of the five lists go into two-level totals.
 *   compact   the create / update / dup / replace / delete lists in index order, with the byte lengths the gathers
 *             need and, with stats, the Stat.version of each update, replace and delete entry's node.
 * Then regk_mkdirp_len_kernel / regk_mkdirp_gather_kernel pack the request sets (create paths and payloads, update
 * paths and payloads, delete paths, replace paths and payloads) into streams of the library's own, which
 * regk_reconcile_requests frames.  Without stats (regk_reconcile) the replace list stays empty.
 *
 * The snapshot may be a caller's device buffer with no slack behind its last byte, so every read of its bytes goes
 * through the clamped helpers of regk_core.cuh (string_word_clamped and friends), which never touch a byte at or past
 * the stream's total; the batch's own streams have >= 16 bytes of slack and use the plain ones.
 */
#ifndef REGK_RECONCILE_CUH
#define REGK_RECONCILE_CUH

#include "regk_kernels.cuh"

namespace regk {

constexpr uint32_t RC_TILE = TILE;              /* items per CTA of the mark / compact passes (128) */
constexpr uint32_t RC_BAD_SLOT = 0xFFFFFFFFu;   /* slot_obs of a node with bad offsets */

enum : uint8_t { RC_SAME = 0, RC_CREATE = 1, RC_UPDATE = 2, RC_DUP = 3, RC_REPLACE = 4 };  /* cls (include/regk.h REGK_DELTA_*) */
enum : uint8_t { RC_KEEP = 0, RC_DELETE = 1 };                               /* obs_cls */
enum { RC_LCREATE, RC_LUPDATE, RC_LDUP, RC_LREPLACE, RC_LDELETE, RC_NLISTS };   /* the record lists first, then the nodes' */
enum { RC_NREC_LISTS = RC_LDELETE };
/* the gathers: create paths / payloads, update paths / payloads, delete paths, replace paths / payloads */
enum { RC_GCREATE = 0, RC_GUPDATE = 2, RC_GDELETE = 4, RC_GREPLACE = 5, RC_NGATHERS = 7 };
enum { RC_VUPDATE, RC_VDELETE, RC_VREPLACE, RC_NVER };                      /* the lists that carry a version */

/* counters[]: [0] smallest node with bad offsets, [1] smallest node with a duplicate path (both ~0 = none, set by the
   host), [2 + list] entries of each list, [7 + k] bytes of gather k */
enum { RC_C_BAD = 0, RC_C_DUPNODE = 1, RC_C_COUNT = 2, RC_C_BYTES = 2 + RC_NLISTS, RC_NCOUNTERS = RC_C_BYTES + RC_NGATHERS };

struct ReconcileParams {
    uint64_t n, m;
    /* desired: the batch finished last (the library's streams) */
    const uint8_t *d_path;
    const unsigned long long *d_path_off;       /* [n + 1] */
    const uint8_t *d_json;
    const unsigned long long *d_json_off;
    uint64_t d_path_limit, d_json_limit;        /* readable bytes: total + slack */
    /* observed: the snapshot */
    const uint8_t *o_path;
    const unsigned long long *o_path_off;       /* [m + 1] */
    const uint8_t *o_json;
    const unsigned long long *o_json_off;
    uint64_t o_path_total, o_json_total;        /* readable bytes: exactly these */
    uint32_t validate;                          /* device snapshot: check the offsets in the insert pass */
    /* the snapshot's Stat (regk_reconcile_owned), NULL for regk_reconcile */
    const int32_t *o_version;                   /* [m] */
    const long long *o_owner;                   /* [m] ephemeral owner, 0 = persistent */
    long long want;                             /* the owner every matched node must have */
    uint32_t mask_o, mask_d;                    /* slots - 1 of T_o / T_d (powers of two) */
    uint32_t *t_obs;                            /* T_o: node + 1, 0 = empty (zeroed by the host) */
    uint32_t *t_des;                            /* T_d: record + 1 */
    uint32_t *slot_obs;                         /* [m] T_o slot of node j, RC_BAD_SLOT for bad offsets */
    uint32_t *hash_obs;                         /* [m] path hash of node j (probes T_d in the mark pass) */
    uint32_t *slot_des;                         /* [n] T_d slot of record i */
    uint8_t *cls;                               /* [n] */
    unsigned long long *match;                  /* [n] */
    uint8_t *obs_cls;                           /* [m] */
    uint32_t *tile_total[RC_NLISTS];            /* records: [ntiles_r], delete: [ntiles_o] */
    unsigned long long *super_total[RC_NLISTS];
    unsigned long long *list[RC_NLISTS];        /* ascending indices */
    uint32_t *len[RC_NGATHERS];                 /* per list entry: the bytes of its path / payload in each gather */
    int32_t *ver[RC_NVER];                      /* per update / delete / replace entry: its node's version (with stats) */
    unsigned long long *counters;               /* [RC_NCOUNTERS] */
    uint32_t tiles_r;                           /* CTAs of the mark / compact passes that cover records; the rest cover nodes */
};

__device__ __forceinline__ uint32_t rc_obs_len(const unsigned long long *off, uint64_t j)
{
    return (uint32_t)(off[j + 1] - off[j]);
}

/* ---- insert: offsets check, then the snapshot's paths into T_o.  (256, 4) here and in the desired pass: with no
   minimum, ptxas for sm_90a keeps these two at 32 / 40 registers and spills; with a 64-register bound they use 39
   and do not. ---- */
__global__ void __launch_bounds__(256, 4) regk_reconcile_insert_kernel(const ReconcileParams p)
{
    const uint64_t j = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (j >= p.m)
        return;
    const unsigned long long o0 = p.o_path_off[j], o1 = p.o_path_off[j + 1];
    if (p.validate) {
        const unsigned long long q0 = p.o_json_off[j], q1 = p.o_json_off[j + 1];
        if (o0 > o1 || o1 > p.o_path_total || o1 - o0 > 0xFFFFFFFFull || q0 > q1 || q1 > p.o_json_total ||
            q1 - q0 > 0xFFFFFFFFull) {
            atomicMin(p.counters + RC_C_BAD, (unsigned long long)j);
            p.slot_obs[j] = RC_BAD_SLOT;
            return;
        }
    }
    const uint32_t *W = reinterpret_cast<const uint32_t *>(p.o_path);
    const uint32_t len = (uint32_t)(o1 - o0);
    const uint32_t h = string_hash32_clamped(W, o0, len, p.o_path_total);
    p.hash_obs[j] = h;
    uint32_t slot = h & p.mask_o;
    for (;;) {
        uint32_t cur = p.t_obs[slot];
        if (cur == 0u) {
            cur = atomicCAS(p.t_obs + slot, 0u, (uint32_t)j + 1u);
            if (cur == 0u)
                break;                                      /* claimed */
        }
        const uint64_t k = cur - 1u;                        /* a node inserted before: its offsets were checked */
        if (k == j)
            break;
        const unsigned long long k0 = p.o_path_off[k];
        if (rc_obs_len(p.o_path_off, k) == len && string_equal2(W, o0, p.o_path_total, W, k0, p.o_path_total, len)) {
            if (cur > (uint32_t)j + 1u)
                atomicMin(p.t_obs + slot, (uint32_t)j + 1u);
            break;                                          /* the same path */
        }
        slot = (slot + 1u) & p.mask_o;
    }
    p.slot_obs[j] = slot;
}

/* ---- desired: match against T_o, compare the payload, insert into T_d ---- */
__global__ void __launch_bounds__(256, 4) regk_reconcile_desired_kernel(const ReconcileParams p)
{
    const uint64_t i = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= p.n)
        return;
    const unsigned long long o0 = p.d_path_off[i];
    const uint32_t len = (uint32_t)(p.d_path_off[i + 1] - o0);
    const uint32_t *W = reinterpret_cast<const uint32_t *>(p.d_path);
    const uint32_t *OW = reinterpret_cast<const uint32_t *>(p.o_path);
    const uint32_t h = string_hash32(W, o0, len);
    /* 1. the node with this path: T_o is complete and read-only here */
    unsigned long long match = ~0ull;
    uint8_t c = RC_CREATE;
    if (p.m) {
        uint32_t slot = h & p.mask_o;
        for (;;) {
            const uint32_t cur = p.t_obs[slot];
            if (cur == 0u)
                break;
            const uint64_t k = cur - 1u;
            const unsigned long long k0 = p.o_path_off[k];
            if (rc_obs_len(p.o_path_off, k) == len && string_equal2(W, o0, p.d_path_limit, OW, k0, p.o_path_total, len)) {
                match = k;
                break;
            }
            slot = (slot + 1u) & p.mask_o;
        }
    }
    if (match != ~0ull && p.o_owner && p.o_owner[match] != p.want) {
        c = RC_REPLACE;                                     /* the payload does not matter: the node is created again */
    } else if (match != ~0ull) {
        const unsigned long long q0 = p.d_json_off[i], k0 = p.o_json_off[match];
        const uint32_t jl = (uint32_t)(p.d_json_off[i + 1] - q0);
        const bool same = rc_obs_len(p.o_json_off, match) == jl &&
            string_equal2(reinterpret_cast<const uint32_t *>(p.d_json), q0, p.d_json_limit,
                          reinterpret_cast<const uint32_t *>(p.o_json), k0, p.o_json_total, jl);
        c = same ? RC_SAME : RC_UPDATE;
    }
    p.cls[i] = c;
    p.match[i] = match;
    /* 2. the first occurrence of this path among the records */
    uint32_t slot = h & p.mask_d;
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

/* ---- mark: DUP records; duplicate nodes; KEEP / DELETE; per-tile counts ---- */
__global__ void __launch_bounds__(RC_TILE) regk_reconcile_mark_kernel(const ReconcileParams p)
{
    const bool rec = blockIdx.x < p.tiles_r;
    const uint32_t tile = rec ? blockIdx.x : blockIdx.x - p.tiles_r;
    const uint64_t i = (uint64_t)tile * RC_TILE + threadIdx.x;
    uint32_t f = 0;                                         /* bit k: goes to list k */
    if (rec) {
        if (i < p.n) {
            uint8_t c = p.cls[i];
            if (p.t_des[p.slot_des[i]] != (uint32_t)i + 1u) {
                c = RC_DUP;
                p.cls[i] = c;
            }
            f = c == RC_CREATE ? 1u << RC_LCREATE : c == RC_UPDATE ? 1u << RC_LUPDATE : c == RC_DUP ? 1u << RC_LDUP :
                c == RC_REPLACE ? 1u << RC_LREPLACE : 0u;
        }
    } else if (i < p.m) {
        const uint32_t so = p.slot_obs[i];
        if (so != RC_BAD_SLOT) {
            if (p.t_obs[so] != (uint32_t)i + 1u)
                atomicMin(p.counters + RC_C_DUPNODE, (unsigned long long)i);
            const unsigned long long o0 = p.o_path_off[i];
            const uint32_t len = rc_obs_len(p.o_path_off, i);
            const uint32_t *W = reinterpret_cast<const uint32_t *>(p.d_path);
            const uint32_t *OW = reinterpret_cast<const uint32_t *>(p.o_path);
            bool keep = false;
            uint32_t slot = p.hash_obs[i] & p.mask_d;
            for (;;) {
                const uint32_t cur = p.t_des[slot];
                if (cur == 0u)
                    break;
                const unsigned long long k0 = p.d_path_off[cur - 1u];
                if ((uint32_t)(p.d_path_off[cur] - k0) == len && string_equal2(OW, o0, p.o_path_total, W, k0, p.d_path_limit, len)) {
                    keep = true;
                    break;
                }
                slot = (slot + 1u) & p.mask_d;
            }
            p.obs_cls[i] = keep ? RC_KEEP : RC_DELETE;
            f = keep ? 0u : 1u << RC_LDELETE;
        } else {
            p.obs_cls[i] = RC_DELETE;                       /* never read: the call is refused */
        }
    }
    if (rec) {
        #pragma unroll
        for (int l = RC_LCREATE; l < RC_NREC_LISTS; l++) {
            const uint32_t c = __popc(__ballot_sync(0xFFFFFFFFu, (f >> l) & 1u));
            if ((threadIdx.x & 31u) == 0)
                add_tile_total(p.tile_total[l], p.super_total[l], tile, c);
        }
    } else {
        const uint32_t c = __popc(__ballot_sync(0xFFFFFFFFu, f != 0u));
        if ((threadIdx.x & 31u) == 0)
            add_tile_total(p.tile_total[RC_LDELETE], p.super_total[RC_LDELETE], tile, c);
    }
}

/* ---- compact: every list in index order, the byte lengths of its entries and, with stats, their versions ---- */
__global__ void __launch_bounds__(RC_TILE) regk_reconcile_compact_kernel(const ReconcileParams p)
{
    constexpr uint32_t NL = RC_NREC_LISTS;                  /* lists of a record CTA (a node CTA has one) */
    __shared__ uint32_t s_warp[NL][RC_TILE / 32];
    __shared__ unsigned long long s_base[NL];
    const bool rec = blockIdx.x < p.tiles_r;
    const uint32_t tile = rec ? blockIdx.x : blockIdx.x - p.tiles_r;
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const int l0 = rec ? RC_LCREATE : RC_LDELETE, nl = rec ? (int)NL : 1;
    if (threadIdx.x < 32) {
        for (int l = 0; l < nl; l++) {
            const unsigned long long b = tile_base_from_totals(p.tile_total[l0 + l], p.super_total[l0 + l], tile);
            if (lane == 0)
                s_base[l] = b;
        }
    }
    const uint64_t i = (uint64_t)tile * RC_TILE + threadIdx.x;
    uint32_t l = NL;                                        /* which of this CTA's lists the item goes to (NL: none) */
    if (rec && i < p.n) {
        const uint8_t c = p.cls[i];
        l = c == RC_CREATE ? RC_LCREATE : c == RC_UPDATE ? RC_LUPDATE : c == RC_DUP ? RC_LDUP : c == RC_REPLACE ? RC_LREPLACE : NL;
    } else if (!rec && i < p.m && p.obs_cls[i] == RC_DELETE && p.slot_obs[i] != RC_BAD_SLOT) {
        l = 0;
    }
    uint32_t bal[NL], rank = 0;
    #pragma unroll
    for (int k = 0; k < (int)NL; k++) {
        bal[k] = __ballot_sync(0xFFFFFFFFu, l == (uint32_t)k);
        if (lane == 0)
            s_warp[k][warp] = __popc(bal[k]);
    }
    __syncthreads();
    if (l < NL) {
        rank = __popc(bal[l] & ((1u << lane) - 1u));
        for (uint32_t w = 0; w < warp; w++)
            rank += s_warp[l][w];
    }
    /* the gather of this entry's path (its payload is the next one), and the version list it feeds (-1: none) */
    const int gq = !rec ? RC_GDELETE : l == RC_LCREATE ? RC_GCREATE : l == RC_LUPDATE ? RC_GUPDATE : l == RC_LREPLACE ? RC_GREPLACE : -1;
    const int vq = !rec ? RC_VDELETE : l == RC_LUPDATE ? RC_VUPDATE : l == RC_LREPLACE ? RC_VREPLACE : -1;
    uint32_t lens[2] = {0u, 0u};                            /* path and payload bytes of this entry */
    if (l < NL) {
        const unsigned long long k = s_base[l] + rank;
        p.list[l0 + l][k] = i;
        if (rec && gq >= 0) {
            lens[0] = (uint32_t)(p.d_path_off[i + 1] - p.d_path_off[i]);
            lens[1] = (uint32_t)(p.d_json_off[i + 1] - p.d_json_off[i]);
            p.len[gq][k] = lens[0];
            p.len[gq + 1][k] = lens[1];
        } else if (!rec) {
            lens[0] = rc_obs_len(p.o_path_off, i);
            p.len[RC_GDELETE][k] = lens[0];
        }
        if (p.o_version && vq >= 0)
            p.ver[vq][k] = p.o_version[rec ? p.match[i] : i];
    }
    /* bytes of each gather; a list no lane of the warp feeds is skipped (the test is warp-uniform) */
    #pragma unroll
    for (int q = 0; q < 3; q++) {
        const uint32_t lq = q == 0 ? RC_LCREATE : q == 1 ? RC_LUPDATE : RC_LREPLACE;
        const int gb = q == 0 ? RC_GCREATE : q == 1 ? RC_GUPDATE : RC_GREPLACE;
        if (rec ? bal[lq] == 0u : (q != 0 || bal[0] == 0u))
            continue;
        #pragma unroll
        for (int s = 0; s < 2; s++) {
            if (!rec && s)
                continue;
            unsigned long long v = (l == (rec ? lq : 0u)) ? lens[s] : 0u;
            #pragma unroll
            for (int d = 16; d > 0; d >>= 1)
                v += __shfl_xor_sync(0xFFFFFFFFu, v, d);
            if (lane == 0 && v)
                atomicAdd(p.counters + RC_C_BYTES + (rec ? gb + s : RC_GDELETE), v);
        }
    }
    const uint64_t items = rec ? p.n : p.m;
    if (i + 1 == items) {                                   /* the thread of the last item closes the lists */
        for (int k = 0; k < nl; k++) {
            uint32_t t = 0;
            for (uint32_t w = 0; w < RC_TILE / 32; w++)
                t += s_warp[k][w];
            p.counters[RC_C_COUNT + l0 + k] = s_base[k] + t;
        }
    }
}

}  /* namespace regk */
#endif /* REGK_RECONCILE_CUH */
