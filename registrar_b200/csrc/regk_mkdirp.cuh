/*
 * regk_mkdirp.cuh — the whole mkdirp set of a batch (reference lib/register.js:107-129, setupDirectories:
 * zk.mkdirp(path.dirname(n)) for every node, and mkdirp creates the directory AND every ancestor of it).
 *
 * From the distinct immediate directories that regk_parents.cuh finds (run on buffers of its own), this computes
 * every ancestor prefix once, ordered by (depth, first record whose directory has it as a prefix), so that a parent
 * always precedes its children and the list can be pipelined on one ZooKeeper session.  A directory is (record r,
 * length L) = path_r[0, L) with r the smallest such record.  The passes:
 *
 *   classify   one thread per distinct directory: mkdir_components() (regk_core.cuh) - root, invalid, or its depth;
 *              the invalid ones go to a list of their own, the others seed the level-1 work list {r, 0, seed, -}.
 *   per depth d = 1, 2, ... while the work list is not empty:
 *     insert   one thread per entry: extend the entry's prefix by one component (mkdir_extend, running FNV state
 *              carried in the entry) and insert (r, L) into an open-addressing table of 64-bit slots
 *              ((r + 1) << 32 | L; 0 = empty): atomicCAS claims an empty slot; a slot with the same L whose record
 *              has the same L bytes (compared byte for byte - the hash only picks the slot) is the same directory,
 *              and atomicMin keeps the smaller record.  L must be stored: one record is the representative of
 *              several prefixes, and a shorter prefix of it would otherwise match the slot of a longer one.
 *     mark     an entry is the first occurrence iff the slot still holds its own key; it continues to depth d + 1
 *              iff its prefix is shorter than its directory.  Per-tile counts of both (two-level totals).
 *     split    first occurrences go to dir_rec / dir_len at depth_off[d - 1] + rank, continuing entries to the next
 *              work list - both in entry order, and entries stay in record order, so depth d comes out sorted by
 *              record with no sort.
 *   gather     per tile of directories: byte offsets (two-level totals of the lengths, block scan) and the packed
 *              bytes, written output-stationary as whole 16-byte blocks (byte stores only at a tile's ragged ends).
 *
 * Every pass is a kernel boundary; the host reads two counters per depth to size the next launch.
 */
#ifndef REGK_MKDIRP_CUH
#define REGK_MKDIRP_CUH

#include "regk_kernels.cuh"

namespace regk {

constexpr uint32_t MK_TILE = TILE;              /* items per CTA of the mark / split / gather passes (128) */

struct MkdirpParams {
    const uint8_t *path_bytes;
    const unsigned long long *path_off;         /* [n + 1] */
    const uint32_t *parent_len;                 /* [n] length of each record's directory */
    /* classify: the distinct immediate directories (ascending records) */
    const unsigned long long *unique_first;
    uint64_t n_unique;
    /* the work list of one depth: {record, prefix length, FNV state, table slot} */
    uint4 *list_in;
    uint4 *list_out;
    uint64_t m;                                 /* items of this pass (directories or entries) */
    uint8_t *flags;                             /* [m] bit 0: goes to the A output, bit 1: to the B output */
    uint32_t *tile_a, *tile_b;                  /* [ntiles] */
    unsigned long long *super_a, *super_b;      /* [ntiles / SUPER + 1] */
    unsigned long long *table;                  /* [mask + 1] */
    uint32_t mask;
    unsigned long long *counters;               /* [0] A items, [1] B items, [2] directory bytes (accumulated), [3] entries */
    /* outputs */
    unsigned long long *invalid;                /* classify A */
    unsigned long long *dir_rec;                /* level A, from dir_base */
    uint32_t *dir_len;
    uint64_t dir_base;
};

/* ---- classify: root / invalid / depth of every distinct immediate directory ---- */
__global__ void __launch_bounds__(MK_TILE) regk_mkdirp_classify_kernel(const MkdirpParams p)
{
    const uint64_t u = (uint64_t)blockIdx.x * MK_TILE + threadIdx.x;
    uint32_t depth = 0, f = 0;
    if (u < p.m) {
        const uint64_t r = p.unique_first[u];
        const uint32_t c = mkdir_components(p.path_bytes + p.path_off[r], p.parent_len[r]);
        f = c == MKDIR_INVALID ? 1u : (c ? 2u : 0u);
        depth = c == MKDIR_INVALID ? 0u : c;
        p.flags[u] = (uint8_t)f;
    }
    const uint32_t na = __popc(__ballot_sync(0xFFFFFFFFu, f & 1u)), nb = __popc(__ballot_sync(0xFFFFFFFFu, f >> 1));
    unsigned long long e = depth;
    #pragma unroll
    for (int d = 16; d > 0; d >>= 1)
        e += __shfl_xor_sync(0xFFFFFFFFu, e, d);
    if ((threadIdx.x & 31u) == 0) {
        add_tile_total(p.tile_a, p.super_a, blockIdx.x, na);
        add_tile_total(p.tile_b, p.super_b, blockIdx.x, nb);
        if (e)
            atomicAdd(p.counters + 3, e);                   /* (directory, depth) entries: sizes the table */
    }
}

/* ---- insert: one more component of every entry's prefix, into the table ---- */
__global__ void __launch_bounds__(256) regk_mkdirp_insert_kernel(const MkdirpParams p)
{
    const uint64_t i = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= p.m)
        return;
    uint4 e = p.list_in[i];
    const uint32_t r = e.x;
    const unsigned long long o = p.path_off[r];
    uint32_t h = e.z;
    const uint32_t L = mkdir_extend(p.path_bytes + o, e.y, p.parent_len[r], &h);
    const unsigned long long key = ((unsigned long long)(r + 1u) << 32) | L;
    const uint32_t *W = reinterpret_cast<const uint32_t *>(p.path_bytes);
    uint32_t slot = mkdir_slot_hash(h, L) & p.mask;
    for (;;) {
        unsigned long long cur = p.table[slot];
        if (cur == 0ull) {
            cur = atomicCAS(p.table + slot, 0ull, key);
            if (cur == 0ull)
                break;                                      /* claimed */
        }
        if ((uint32_t)cur == L) {                           /* same length: compare with the slot's record */
            const uint64_t j = (cur >> 32) - 1u;
            if (j == r || string_equal(W, o, p.path_off[j], L)) {
                if (cur > key)                              /* keys of one slot differ only in the record */
                    atomicMin(p.table + slot, key);
                break;
            }
        }
        slot = (slot + 1u) & p.mask;
    }
    p.list_in[i] = make_uint4(r, L, h, slot);
}

/* ---- mark: first occurrence (A) / continues to the next depth (B) ---- */
__global__ void __launch_bounds__(MK_TILE) regk_mkdirp_mark_kernel(const MkdirpParams p)
{
    const uint64_t i = (uint64_t)blockIdx.x * MK_TILE + threadIdx.x;
    uint32_t f = 0;
    if (i < p.m) {
        const uint4 e = p.list_in[i];
        const unsigned long long key = ((unsigned long long)(e.x + 1u) << 32) | e.y;
        f = (p.table[e.w] == key ? 1u : 0u) | (e.y < p.parent_len[e.x] ? 2u : 0u);
        p.flags[i] = (uint8_t)f;
    }
    const uint32_t na = __popc(__ballot_sync(0xFFFFFFFFu, f & 1u)), nb = __popc(__ballot_sync(0xFFFFFFFFu, f >> 1));
    if ((threadIdx.x & 31u) == 0) {
        add_tile_total(p.tile_a, p.super_a, blockIdx.x, na);
        add_tile_total(p.tile_b, p.super_b, blockIdx.x, nb);
    }
}

/* ---- split: items flagged A and B to their outputs, in item order.  LEVEL = false: after classify (A = invalid
   list, B = the depth-1 work list); LEVEL = true: after mark (A = directories of this depth, B = next work list) */
template <bool LEVEL>
__global__ void __launch_bounds__(MK_TILE) regk_mkdirp_split_kernel(const MkdirpParams p)
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
    const uint64_t i = (uint64_t)tile * MK_TILE + threadIdx.x;
    const uint32_t f = i < p.m ? p.flags[i] : 0u;
    const uint32_t ba = __ballot_sync(0xFFFFFFFFu, f & 1u), bb = __ballot_sync(0xFFFFFFFFu, f >> 1);
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
    uint32_t len = 0;
    if (f) {
        if (!LEVEL) {
            const unsigned long long r = p.unique_first[i];
            if (f & 1u)
                p.invalid[s_base[0] + ra] = r;
            if (f & 2u)
                p.list_out[s_base[1] + rb] = make_uint4((uint32_t)r, 0u, MKDIR_HASH_SEED, 0u);
        } else {
            const uint4 e = p.list_in[i];
            if (f & 1u) {
                p.dir_rec[p.dir_base + s_base[0] + ra] = e.x;
                p.dir_len[p.dir_base + s_base[0] + ra] = e.y;
                len = e.y;
            }
            if (f & 2u)
                p.list_out[s_base[1] + rb] = make_uint4(e.x, e.y, e.z, 0u);
        }
    }
    if (LEVEL) {
        unsigned long long bytes = len;
        #pragma unroll
        for (int d = 16; d > 0; d >>= 1)
            bytes += __shfl_xor_sync(0xFFFFFFFFu, bytes, d);
        if (lane == 0 && bytes)
            atomicAdd(p.counters + 2, bytes);
    }
    if (i + 1 == p.m) {                                     /* the thread of the last item closes both lists */
        p.counters[0] = s_base[0] + ta;
        p.counters[1] = s_base[1] + tb;
    }
}

/* ---- gather: dir_off and the packed directory bytes ---- */
struct MkGatherParams {
    uint64_t n_dirs;
    const uint8_t *path_bytes;
    const unsigned long long *path_off;
    const unsigned long long *dir_rec;
    const uint32_t *dir_len;
    unsigned long long *tile_total;             /* [ntiles] bytes of each tile's directories */
    unsigned long long *super_total;            /* [ntiles / SUPER + 1] */
    uint8_t *dir_bytes;
    unsigned long long *dir_off;                /* [n_dirs + 1] */
};

__global__ void __launch_bounds__(MK_TILE) regk_mkdirp_len_kernel(const MkGatherParams p)
{
    __shared__ unsigned long long s_warp[MK_TILE / 32];
    const uint64_t k = (uint64_t)blockIdx.x * MK_TILE + threadIdx.x;
    unsigned long long v = k < p.n_dirs ? p.dir_len[k] : 0u;
    #pragma unroll
    for (int d = 16; d > 0; d >>= 1)
        v += __shfl_xor_sync(0xFFFFFFFFu, v, d);
    if ((threadIdx.x & 31u) == 0)
        s_warp[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long t = 0;
        for (uint32_t w = 0; w < MK_TILE / 32; w++)
            t += s_warp[w];
        p.tile_total[blockIdx.x] = t;
        if (t)
            atomicAdd(p.super_total + blockIdx.x / SUPER, t);
    }
}

__global__ void __launch_bounds__(MK_TILE) regk_mkdirp_gather_kernel(const MkGatherParams p)
{
    __shared__ unsigned long long s_warp[MK_TILE / 32];
    __shared__ unsigned long long s_off[MK_TILE + 1];           /* tile-relative byte offsets */
    __shared__ unsigned long long s_src[MK_TILE];               /* where each directory's bytes start in the path stream */
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
    const uint32_t nd = (uint32_t)min((uint64_t)MK_TILE, p.n_dirs - k0);
    const unsigned long long len = threadIdx.x < nd ? p.dir_len[k] : 0ull;
    if (threadIdx.x < nd)
        s_src[threadIdx.x] = p.path_off[p.dir_rec[k]];
    unsigned long long total;
    const unsigned long long excl = block_scan<unsigned long long>(s_warp, len, &total);   /* barriers: s_base, s_src */
    const unsigned long long base = s_base;
    if (threadIdx.x < nd) {
        s_off[threadIdx.x] = excl;
        p.dir_off[k] = base + excl;
    }
    if (threadIdx.x == 0)
        s_off[nd] = total;
    if (k0 + nd == p.n_dirs && threadIdx.x == 0)
        p.dir_off[p.n_dirs] = base + total;
    __syncthreads();
    /* output-stationary: every 16-byte block of [base, base + total) that this tile owns, assembled in registers */
    const unsigned long long a0 = base & ~15ull;
    const uint32_t lead = (uint32_t)(base - a0);
    const unsigned long long nblk = (lead + total + 15ull) >> 4;
    for (unsigned long long b = threadIdx.x; b < nblk; b += MK_TILE) {
        const long long bs = (long long)(16ull * b) - (long long)lead;   /* tile-relative byte of the block's lane 0 */
        const unsigned long long pos0 = bs < 0 ? 0ull : (unsigned long long)bs;
        const unsigned long long end = min((unsigned long long)(bs + 16), total);
        uint32_t lo = 0, hi = nd - 1u;                          /* the directory pos0 lies in: last s_off[d] <= pos0 */
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
            const uint32_t byte = p.path_bytes[s_src[d] + (q - s_off[d])];
            const uint32_t lanebyte = (uint32_t)(q - (unsigned long long)bs);
            acc[lanebyte >> 2] |= byte << (8u * (lanebyte & 3u));
        }
        uint8_t *gp = p.dir_bytes + a0 + 16ull * b;
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

}  /* namespace regk */
#endif /* REGK_MKDIRP_CUH */
