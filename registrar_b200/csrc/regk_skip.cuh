/*
 * regk_skip.cuh — skip mode (REGK_SKIP_BAD): the redo of a batch in which some records failed the value fence.
 *
 * The compose kernels only report THAT a batch has out-of-domain records (OR of the bits, smallest index).  When
 * a skip-mode batch comes back dirty, regk_finish runs three passes around an ordinary second run:
 *   1. regk_fence_kernel    one thread per record: fence_record() (regk_core.cuh) -> bits[i], and per-tile totals
 *                           over the KEPT records of five quantities (records, domain bytes, variable-length host
 *                           bytes, address bytes, port elements) in the two-level tile / super-tile layout
 *   2. regk_compact_kernel  one CTA per tile: the kept records' fields -> a library-owned regk_batch with u32
 *                           offsets (the batch of the kept records alone), their bytes moved run by run (runs of
 *                           consecutive kept records) with 16-byte stores; the skipped ones -> an ascending index
 *                           list (slot of skipped record i = i - kept_before(i))
 *      ... regk_register_batch on that batch (device in, device out; the exact-offset redo included) ...
 *   3. regk_expand_kernel   off[i] = compacted_off[kept_before(i)] for i in [0, n]: a skipped record gets an empty
 *                           path and payload, and the compacted byte streams are the result's streams
 * A clean skip-mode batch never reaches this file: it runs exactly the kernels of a plain batch.
 */
#ifndef REGK_SKIP_CUH
#define REGK_SKIP_CUH

#include "regk_kernels.cuh"

namespace regk {

enum : int { SKIP_REC = 0, SKIP_DOM, SKIP_HOST, SKIP_ADDR, SKIP_PORTS, SKIP_Q };

struct SkipStatus {
    uint32_t bad_bits;                          /* OR over the batch */
    uint32_t pad;
    unsigned long long first_bad;               /* bitwise NOT of the smallest offending index (as DevStatus) */
    unsigned long long total[SKIP_Q];           /* kept records and their bytes / port elements */
};

struct SkipParams {
    uint64_t n;
    uint32_t alias, do_path, do_json, ntypes;
    /* the batch as its compose kernels read it (device) */
    const uint8_t *domain_bytes;
    const uint32_t *domain_off;
    const uint8_t *host_bytes;
    const uint32_t *host_off;                   /* NULL: fixed stride */
    uint32_t host_stride;
    const uint8_t *type_id;
    const uint8_t *addr_bytes;
    const uint32_t *addr_off;
    const int32_t *ttl;
    const uint32_t *ports_off;
    const uint32_t *ports;
    const uint8_t *ports_present;
    /* workspace */
    uint8_t *bits;                              /* [n] REGK_BAD_* of every record */
    uint32_t *tile_total[SKIP_Q];               /* [ntiles] each */
    unsigned long long *super_total[SKIP_Q];    /* [ntiles / SUPER + 1] each */
    SkipStatus *status;
    /* the compacted batch (NULL where the source array is NULL or not needed) */
    uint8_t *c_domain_bytes;
    uint32_t *c_domain_off;
    uint8_t *c_host_bytes;
    uint32_t *c_host_off;
    uint8_t *c_type_id;
    uint8_t *c_addr_bytes;
    uint32_t *c_addr_off;
    int32_t *c_ttl;
    uint32_t *c_ports_off;
    uint32_t *c_ports;
    uint8_t *c_ports_present;
    unsigned long long *skip_index;             /* [n - kept] */
    uint8_t *skip_bits;                         /* [n - kept] */
};

/* the fields of record r the compaction moves */
struct SkipRec {
    uint32_t d0, L, h0, H, a0, al, p0, k;
};

__device__ __forceinline__ SkipRec skip_rec(const SkipParams &p, uint64_t r)
{
    SkipRec x{};
    if (p.do_path) {
        x.d0 = p.domain_off[r];
        x.L = p.domain_off[r + 1] - x.d0;
        if (!p.alias) {
            if (p.host_off) {
                x.h0 = p.host_off[r];
                x.H = p.host_off[r + 1] - x.h0;
            } else {
                x.h0 = 0;
                x.H = p.host_stride;
            }
        }
    }
    if (p.do_json) {
        x.a0 = p.addr_off[r];
        x.al = p.addr_off[r + 1] - x.a0;
        if (p.ports_off) {
            x.p0 = p.ports_off[r];
            x.k = p.ports_off[r + 1] - x.p0;
        }
    }
    return x;
}

/* warp sums of the five quantities -> the tile's two-level totals and the batch totals */
__device__ __forceinline__ void skip_add_totals(const SkipParams &p, uint32_t tile, uint32_t (&q)[SKIP_Q])
{
    #pragma unroll
    for (int j = 0; j < SKIP_Q; j++) {
        #pragma unroll
        for (int d = 16; d > 0; d >>= 1)
            q[j] += __shfl_xor_sync(0xFFFFFFFFu, q[j], d);
    }
    if ((threadIdx.x & 31u) == 0) {
        #pragma unroll
        for (int j = 0; j < SKIP_Q; j++) {
            add_tile_total(p.tile_total[j], p.super_total[j], tile, q[j]);
            if (q[j])
                atomicAdd(&p.status->total[j], (unsigned long long)q[j]);
        }
    }
}

/* 1. fence pass.  Offsets are trusted: the batch reached this pass only without REGK_BAD_TOO_LARGE. */
__global__ void __launch_bounds__(TILE) regk_fence_kernel(const SkipParams p)
{
    const uint32_t tile = blockIdx.x, t = threadIdx.x;
    const uint64_t r0 = (uint64_t)tile * TILE, r = r0 + t;
    uint32_t q[SKIP_Q] = {0, 0, 0, 0, 0};
    if (r < p.n) {
        const SkipRec x = skip_rec(p, r);
        /* fixed-stride hostnames are addressed from the tile's first one (a multiple of 128 strides: word aligned) */
        const uint8_t *hbase = p.host_off ? p.host_bytes : p.host_bytes + r0 * p.host_stride;
        const uint32_t h0 = p.host_off ? x.h0 : t * p.host_stride;
        const uint32_t bad = fence_record(GuardedWords{reinterpret_cast<const uint32_t *>(p.domain_bytes)}, x.d0, x.L,
            GuardedWords{reinterpret_cast<const uint32_t *>(hbase)}, h0, x.H,
            GuardedWords{reinterpret_cast<const uint32_t *>(p.addr_bytes)}, x.a0, x.al,
            p.do_json ? (uint32_t)p.type_id[r] : 0u, p.ntypes, p.alias != 0, p.do_path != 0, p.do_json != 0);
        p.bits[r] = (uint8_t)bad;
        if (bad) {
            atomicOr(&p.status->bad_bits, bad);
            atomicMax(&p.status->first_bad, ~(unsigned long long)r);
        } else {
            q[SKIP_REC] = 1;
            q[SKIP_DOM] = x.L;
            q[SKIP_HOST] = p.host_off ? x.H : 0u;
            q[SKIP_ADDR] = x.al;
            q[SKIP_PORTS] = x.k;
        }
    }
    skip_add_totals(p, tile, q);
}

/* CTA-cooperative copy of len bytes: aligned 16-byte stores over the destination, the source read as words and
   realigned with funnel shifts; the partial blocks at either end go byte by byte.  Not inlined: inlined into
   regk_compact_kernel's four call sites it made ptxas spill */
__device__ __noinline__ void cta_copy(uint8_t *dst, const uint8_t *src, uint64_t len)
{
    if (len == 0)
        return;
    const uint32_t t = threadIdx.x;
    const uintptr_t d0 = (uintptr_t)dst, a0 = (d0 + 15u) & ~(uintptr_t)15, a1 = (d0 + len) & ~(uintptr_t)15;
    if (a0 >= a1) {
        for (uint64_t i = t; i < len; i += TILE)
            dst[i] = src[i];
        return;
    }
    const uint64_t head = a0 - d0, body_end = a1 - d0;
    for (uint64_t i = t; i < head; i += TILE)
        dst[i] = src[i];
    for (uint64_t i = body_end + t; i < len; i += TILE)
        dst[i] = src[i];
    const uint32_t sh = (uint32_t)(((uintptr_t)src + head) & 3u) * 8u;
    for (uint64_t b = head + 16ull * t; b < body_end; b += 16ull * TILE) {
        const uint32_t *w = reinterpret_cast<const uint32_t *>(((uintptr_t)src + b) & ~(uintptr_t)3);
        uint4 v;
        if (sh == 0) {
            v = make_uint4(w[0], w[1], w[2], w[3]);
        } else {                                                /* the fifth word holds the block's last bytes */
            const uint32_t w0 = w[0], w1 = w[1], w2 = w[2], w3 = w[3], w4 = w[4];
            v = make_uint4(funnel_r(w0, w1, sh), funnel_r(w1, w2, sh), funnel_r(w2, w3, sh), funnel_r(w3, w4, sh));
        }
        *reinterpret_cast<uint4 *>(dst + b) = v;
    }
}

/* 2. compaction: one CTA per tile.  Each thread writes its kept record's per-record fields; the byte ranges move
   as whole runs of consecutive kept records (the whole tile when nothing in it was skipped) by cta_copy. */
__global__ void __launch_bounds__(TILE) regk_compact_kernel(const SkipParams p)
{
    __shared__ uint32_t warp_sum[WARPS];
    __shared__ unsigned long long s_base[SKIP_Q];
    __shared__ uint32_t s_local[SKIP_Q][TILE + 1];              /* per kept record: its place among the tile's kept */
    __shared__ uint8_t s_skip[TILE];                            /* local indices of the skipped records, ascending */
    const uint32_t tile = blockIdx.x, t = threadIdx.x;
    const uint64_t r0 = (uint64_t)tile * TILE;
    const uint32_t nrec = (uint32_t)min((uint64_t)TILE, p.n - r0);
    const bool live = t < nrec;
    const uint64_t r = r0 + (live ? t : 0u);
    if (t < 32) {
        #pragma unroll
        for (int j = 0; j < SKIP_Q; j++) {
            const unsigned long long b = tile_base_from_totals(p.tile_total[j], p.super_total[j], tile);
            if (t == 0)
                s_base[j] = b;
        }
    }
    const uint32_t bad = live ? p.bits[r] : 0u;
    const bool keep = live && bad == 0;
    const SkipRec x = skip_rec(p, r);
    const bool var_host = p.host_off != nullptr;
    uint32_t tot[SKIP_Q], l[SKIP_Q];
    l[SKIP_REC] = block_scan<uint32_t>(warp_sum, keep ? 1u : 0u, &tot[SKIP_REC]);   /* its barriers publish s_base */
    l[SKIP_DOM] = block_scan<uint32_t>(warp_sum, keep ? x.L : 0u, &tot[SKIP_DOM]);
    l[SKIP_HOST] = block_scan<uint32_t>(warp_sum, keep && var_host ? x.H : 0u, &tot[SKIP_HOST]);
    l[SKIP_ADDR] = block_scan<uint32_t>(warp_sum, keep ? x.al : 0u, &tot[SKIP_ADDR]);
    l[SKIP_PORTS] = block_scan<uint32_t>(warp_sum, keep ? x.k : 0u, &tot[SKIP_PORTS]);
    const unsigned long long b_rec = s_base[SKIP_REC], b_dom = s_base[SKIP_DOM], b_host = s_base[SKIP_HOST],
                             b_addr = s_base[SKIP_ADDR], b_ports = s_base[SKIP_PORTS];
    const uint64_t c = b_rec + l[SKIP_REC];                     /* kept_before(r) */
    #pragma unroll
    for (int j = 0; j < SKIP_Q; j++)
        s_local[j][t] = l[j];
    if (live && !keep) {
        p.skip_index[r - c] = r;
        p.skip_bits[r - c] = (uint8_t)bad;
        s_skip[t - l[SKIP_REC]] = (uint8_t)t;
    }
    if (keep) {
        if (p.do_path) {
            p.c_domain_off[c] = (uint32_t)(b_dom + l[SKIP_DOM]);
            if (!p.alias && var_host)
                p.c_host_off[c] = (uint32_t)(b_host + l[SKIP_HOST]);
        }
        if (p.do_json) {
            p.c_type_id[c] = p.type_id[r];
            p.c_addr_off[c] = (uint32_t)(b_addr + l[SKIP_ADDR]);
            if (p.ttl)
                p.c_ttl[c] = p.ttl[r];
            if (p.ports_off)
                p.c_ports_off[c] = (uint32_t)(b_ports + l[SKIP_PORTS]);
            if (p.ports_present)
                p.c_ports_present[c] = p.ports_present[r];
        }
    }
    __syncthreads();                                            /* s_local / s_skip published */
    const uint32_t nskip = nrec - tot[SKIP_REC];
    for (uint32_t k = 0; k <= nskip; k++) {                     /* run k: the kept records between skips k-1 and k */
        const uint32_t a = k ? s_skip[k - 1] + 1u : 0u, e = k < nskip ? (uint32_t)s_skip[k] : nrec;
        if (a >= e)
            continue;
        const uint64_t ra = r0 + a, re = r0 + e;
        if (p.do_path) {
            cta_copy(p.c_domain_bytes + b_dom + s_local[SKIP_DOM][a], p.domain_bytes + p.domain_off[ra],
                p.domain_off[re] - p.domain_off[ra]);
            if (!p.alias) {
                if (var_host)
                    cta_copy(p.c_host_bytes + b_host + s_local[SKIP_HOST][a], p.host_bytes + p.host_off[ra],
                        p.host_off[re] - p.host_off[ra]);
                else
                    cta_copy(p.c_host_bytes + (b_rec + s_local[SKIP_REC][a]) * p.host_stride, p.host_bytes + ra * p.host_stride,
                        (uint64_t)(e - a) * p.host_stride);
            }
        }
        if (p.do_json) {
            cta_copy(p.c_addr_bytes + b_addr + s_local[SKIP_ADDR][a], p.addr_bytes + p.addr_off[ra],
                p.addr_off[re] - p.addr_off[ra]);
            if (p.ports_off)
                cta_copy(reinterpret_cast<uint8_t *>(p.c_ports + b_ports + s_local[SKIP_PORTS][a]),
                    reinterpret_cast<const uint8_t *>(p.ports + p.ports_off[ra]), 4ull * (p.ports_off[re] - p.ports_off[ra]));
        }
    }
    if (r0 + nrec == p.n && t == 0) {                           /* closing entries of the compacted offsets */
        const uint64_t kept = b_rec + tot[SKIP_REC];
        if (p.do_path) {
            p.c_domain_off[kept] = (uint32_t)(b_dom + tot[SKIP_DOM]);
            if (!p.alias && var_host)
                p.c_host_off[kept] = (uint32_t)(b_host + tot[SKIP_HOST]);
        }
        if (p.do_json) {
            p.c_addr_off[kept] = (uint32_t)(b_addr + tot[SKIP_ADDR]);
            if (p.ports_off)
                p.c_ports_off[kept] = (uint32_t)(b_ports + tot[SKIP_PORTS]);
        }
    }
}

/* 3. offset expansion over n + 1 entries: off[i] = c_off[kept_before(i)] (either pair may be NULL) */
struct ExpandParams {
    uint64_t n;
    const uint8_t *bits;
    const uint32_t *tile_total;                 /* kept records per tile (the fence pass's SKIP_REC totals) */
    const unsigned long long *super_total;
    const unsigned long long *c_path_off, *c_json_off;
    unsigned long long *path_off, *json_off;
};

__global__ void __launch_bounds__(TILE) regk_expand_kernel(const ExpandParams p)
{
    __shared__ uint32_t warp_sum[WARPS];
    __shared__ unsigned long long s_base;
    const uint32_t tile = blockIdx.x, t = threadIdx.x;
    const uint64_t r = (uint64_t)tile * TILE + t;
    if (t < 32) {
        const unsigned long long b = tile_base_from_totals(p.tile_total, p.super_total, tile);
        if (t == 0)
            s_base = b;
    }
    const bool keep = r < p.n && p.bits[r] == 0;
    uint32_t tot;
    const uint32_t local = block_scan<uint32_t>(warp_sum, keep ? 1u : 0u, &tot);
    if (r <= p.n) {                                             /* entry n: kept_before(n) = all kept records */
        const uint64_t c = s_base + local;
        if (p.c_path_off)
            p.path_off[r] = p.c_path_off[c];
        if (p.c_json_off)
            p.json_off[r] = p.c_json_off[c];
    }
}

}  /* namespace regk */

#endif
