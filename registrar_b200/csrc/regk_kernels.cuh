/*
 * regk_kernels.cuh — sm_90a kernels of the registration hot path.
 *
 *   regk_path_kernel   A1/A2 + A5: domain -> reversed-label znode path (+ '/' + hostname),
 *                      fused with the prefix scan that places every record in the packed
 *                      output stream (lib/register.js:34-39, :221-223)
 *   regk_json_kernel   A3/A4 + A5: host-record JSON payload bytes (lib/register.js:141-159)
 *
 * Shape shared by both (HBM-bound byte work, no tensor cores):
 *   - one CTA = one tile of TILE consecutive records, one thread = one record; tiles
 *     are fully independent (no inter-CTA dependency, no spinning):
 *       * path offsets are closed-form in the input offsets whenever no label is empty
 *         (path_len = L + 2 + H, so path_off[i] = domain_off[i] + host_pos(i) + 2i); the
 *         kernel verifies this against the exact length it derives from the dot bitmap and
 *         raises `needs_exact` otherwise, in which case the host re-runs the batch through
 *         regk_path_len_kernel (exact lengths + last-block scan) and this kernel again;
 *       * payload lengths depend on the values (digits of ttl / ports), so a light
 *         metadata-only pre-kernel (regk_json_len_kernel) produces per-tile totals and
 *         its last CTA scans them into per-tile bases;
 *     (a first version fused a decoupled look-back scan into these kernels: with ~35 KB
 *     tiles the chain's per-window latency capped throughput at ~38 tiles/us = 1.2 TB/s,
 *     33-39 % of all stall samples sat at the barrier behind the look-back —
 *     profiles/r1_lookback_*.txt);
 *   - inputs of the tile are staged into shared memory with 16-byte coalesced loads
 *     (the packed byte streams are contiguous per tile);
 *   - a cooperative, vectorised pre-pass lower-cases the staged domain bytes, builds a
 *     one-bit-per-byte "is '.'" bitmap and applies the input fence;
 *   - records are composed word-wise into a shared-memory image of the tile's output
 *     range, laid out with the same 16-byte phase as the global destination, and
 *     flushed with 16-byte coalesced stores;
 *   - tiles whose bytes do not fit the shared-memory budget take a generic path
 *     (same composers, global-memory source, byte sink) — still on the GPU.
 */
#ifndef REGK_KERNELS_CUH
#define REGK_KERNELS_CUH

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/regk.h"
#include "regk_core.cuh"

namespace regk {

#ifndef REGK_TILE
#define REGK_TILE 128
#endif
/*
 * Minimum resident CTAs per SM for the compose kernels' __launch_bounds__, which sets their register cap
 * (65536 / (TILE * MINB), rounded down to a multiple of 8).  Shared memory, not registers, decides how many CTAs
 * fit: a path tile of config 3 or 5 needs about 26 KB, so at most 8 fit in the SM's 228 KB.  The payload kernel's
 * image and fragment table take about 19 KB, so at most 11 fit.  A cap of 12 (40 registers) made both kernels
 * spill and bought no occupancy on those workloads.  8 gives the path kernel 64 registers and 10 gives the payload
 * kernel 48, and neither spills.  On an H100 SXM, that cut the config 3 step by 2.5 % (DESIGN.md §4).
 */
#ifndef REGK_MINB_PATH
#define REGK_MINB_PATH 8
#endif
#ifndef REGK_MINB_JSON
#define REGK_MINB_JSON 10
#endif
constexpr int TILE = REGK_TILE;                 /* records per tile == threads per CTA */
constexpr int WARPS = TILE / 32;

/* device-side run status, copied to the host after the kernels */
struct DevStatus {
    uint32_t bad_bits;
    uint32_t overflow;                          /* output capacity exceeded (internal error) */
    unsigned long long first_bad;               /* bitwise NOT of the smallest offending record index */
    unsigned long long path_total;
    unsigned long long json_total;
    uint32_t needs_exact;                       /* a record had empty labels: closed-form path offsets do not hold */
    uint32_t generic_tiles;                     /* tiles (of either kernel) whose bytes did not fit the shared-memory budget */
};

__device__ __forceinline__ uint4 ldg_nc_v4(const void *p)
{
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}

__device__ __forceinline__ void stg_v4(void *p, const uint4 &v)
{
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};"
                 ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

/* ---- TMA bulk copy + mbarrier primitives (SASS UBLKCP / SYNCS) ---- */
__device__ __forceinline__ uint32_t smem_u32(const void *p)
{
    return (uint32_t)__cvta_generic_to_shared(p);
}

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}

__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
    uint32_t done;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    } while (!done);
}

/*
 * Manual staging (only for the last blocks of a stream, where whole 16-byte blocks would reach past the
 * caller's buffer): global byte range [g0, g1) of `src` (16-byte aligned base) -> shared memory so that
 * global byte g lands at smem byte g - (g0 & ~15); bytes at or past `limit` are not touched (zero filled).
 */
__device__ __forceinline__ void stage_in(uint8_t *smem, const uint8_t *src, uint64_t g0, uint64_t g1,
    uint64_t limit)
{
    const uint64_t a0 = g0 & ~15ull;
    const uint8_t *base = src + a0;
    const uint32_t nchunks = (uint32_t)((g1 - a0 + 15) >> 4);
    const uint32_t safe = limit > a0 ? (uint32_t)min((uint64_t)nchunks, (limit - a0) >> 4) : 0u;   /* fully inside the buffer */
    for (uint32_t c = threadIdx.x; c < nchunks; c += TILE) {
        if (c < safe) {
            reinterpret_cast<uint4 *>(smem)[c] = ldg_nc_v4(base + 16u * c);
        } else {
            for (uint32_t k = 0; k < 16; k++)
                smem[16u * c + k] = (a0 + 16ull * c + k < limit) ? base[16u * c + k] : (uint8_t)0;
        }
    }
}

/*
 * Flush the shared-memory image of the tile's output range to global memory.
 * smem byte i corresponds to global byte (gbase & ~15) + i; valid bytes are
 * [gbase, gbase + total).  The 16-byte-aligned body goes out as ONE bulk
 * asynchronous copy (cp.async.bulk shared::cta -> global, the TMA engine; SASS
 * UBLKCP) issued by a single thread; the < 16-byte head and tail are stored
 * byte-wise by the first 48 threads.  Callers must have executed fence_proxy_async() after
 * their shared-memory writes and a block barrier before calling.
 */
__device__ __forceinline__ void fence_proxy_async()
{
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

__device__ __forceinline__ void flush_out(uint8_t *gout, const uint8_t *smem, uint64_t gbase, uint32_t total)
{
    const uint64_t a0 = gbase & ~15ull;
    const uint32_t lo = (uint32_t)(gbase - a0);
    const uint32_t hi = lo + total;
    uint32_t body_lo = (lo + 15u) & ~15u, body_hi = hi & ~15u;
    if (body_hi <= body_lo)
        body_lo = body_hi = hi;                 /* nothing aligned: everything is "head" */
    const uint32_t t = threadIdx.x;
    if (t == 0 && body_hi > body_lo) {
        const uint32_t src = (uint32_t)__cvta_generic_to_shared(smem + body_lo);
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                     ::"l"(gout + a0 + body_lo), "r"(src), "r"(body_hi - body_lo) : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
    if (t < 32) {                               /* head: < 16 bytes, or all of a span with no aligned block (< 31) */
        const uint32_t i = lo + t;
        if (i < body_lo)
            gout[a0 + i] = smem[i];
    } else if (t < 48) {                        /* tail: < 16 bytes */
        const uint32_t i = body_hi + (t - 32);
        if (i < hi)
            gout[a0 + i] = smem[i];
    }
    if (t == 0 && body_hi > body_lo)            /* shared memory must stay alive until the engine has read it */
        asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}

/*
 * ---- multi-GPU job: extra destinations of a tile (include/regk.h regk_job) ----
 * A rank's compose kernels place their output directly at its final position in the WHOLE-JOB stream
 * (out_bytes = the rank's own whole-job buffer, offsets biased by the bytes of the ranks before it) and, when
 * `PeerDst::n` > 0, store every tile a second, third ... time into the same position of the peers' whole-job
 * buffers (CUDA-IPC mapped, so a store travels over NVLink / NVSwitch): the all-gather is fused into the
 * compose kernels tile by tile, straight out of shared memory, and no rank ever re-reads its shard from HBM.
 */
struct PeerDst {
    uint32_t n;                                     /* number of extra destinations (0: single-GPU behaviour) */
    uint32_t job;                                   /* 1: output positions are job-absolute (see kernels) */
    uint8_t *bytes[REGK_MAX_PEERS - 1];             /* the peers' whole-job byte buffers (16-byte aligned) */
    unsigned long long *off[REGK_MAX_PEERS - 1];    /* the peers' offset arrays, already advanced to this rank's first record */
};

/* parameter arrays cannot be indexed dynamically without a local-memory copy of the whole block: lanes pick
   their entry with compile-time indices and park it in shared memory */
__device__ __forceinline__ void peer_tables(const PeerDst &pd, uint8_t **s_pb, unsigned long long **s_po)
{
    const uint32_t t = threadIdx.x;
    if (t < REGK_MAX_PEERS - 1) {
        uint8_t *b = nullptr;
        unsigned long long *o = nullptr;
        #pragma unroll
        for (int q = 0; q < REGK_MAX_PEERS - 1; q++)
            if (t == (uint32_t)q) {
                b = pd.bytes[q];
                o = pd.off[q];
            }
        s_pb[t] = b;
        s_po[t] = o;
    }
}

/* bytes [lo, hi) of one 16-byte block of the image (0 <= lo < hi <= 16), stored with the widest naturally aligned
   stores that stay inside the range (at most six): the other bytes of the block belong to the neighbouring tile */
__device__ __forceinline__ void store_block_part(uint8_t *gblk, const uint8_t *sblk, uint32_t lo, uint32_t hi)
{
    while (lo < hi) {
        const uint32_t left = hi - lo;
        if (!(lo & 7u) && left >= 8u) {
            *reinterpret_cast<uint64_t *>(gblk + lo) = *reinterpret_cast<const uint64_t *>(sblk + lo);
            lo += 8u;
        } else if (!(lo & 3u) && left >= 4u) {
            *reinterpret_cast<uint32_t *>(gblk + lo) = *reinterpret_cast<const uint32_t *>(sblk + lo);
            lo += 4u;
        } else if (!(lo & 1u) && left >= 2u) {
            *reinterpret_cast<uint16_t *>(gblk + lo) = *reinterpret_cast<const uint16_t *>(sblk + lo);
            lo += 2u;
        } else {
            gblk[lo] = sblk[lo];
            lo += 1u;
        }
    }
}

__device__ __forceinline__ void bulk_s2g(uint8_t *gdst, const uint8_t *smem_src, uint32_t bytes)
{
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                 ::"l"(gdst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
}

/*
 * flush_out for a job tile: the image goes to the rank's own buffer AND to every peer, all issued by one thread:
 * per destination one bulk copy of the aligned body by the TMA engine, and the ragged head and tail blocks stored
 * piecewise with aligned 8/4/2/1-byte stores (the neighbouring tiles, possibly of another rank, own the other
 * bytes of those blocks; Hopper's bulk copy has no byte mask).  Same preconditions as flush_out.
 */
__device__ __forceinline__ void flush_out_job(uint8_t *gout, uint8_t *const *s_pb, uint32_t npeers, const uint8_t *smem,
    uint64_t gbase, uint32_t total)
{
    if (threadIdx.x != 0 || total == 0)
        return;
    const uint64_t a0 = gbase & ~15ull;
    const uint32_t lo = (uint32_t)(gbase - a0);
    const uint32_t hi = lo + total;
    const uint32_t b_first = lo >> 4, b_last = (hi - 1u) >> 4;          /* 16-byte blocks of the image that hold bytes */
    for (uint32_t d = 0; d <= npeers; d++) {
        uint8_t *g = (d == 0 ? gout : s_pb[d - 1]) + a0;
        if (b_first == b_last) {
            store_block_part(g + 16u * b_first, smem + 16u * b_first, lo & 15u, ((hi - 1u) & 15u) + 1u);
        } else {
            uint32_t body_lo = lo, body_hi = hi;
            if (lo & 15u) {
                store_block_part(g + 16u * b_first, smem + 16u * b_first, lo & 15u, 16u);
                body_lo = 16u * (b_first + 1u);
            }
            if (hi & 15u) {
                store_block_part(g + 16u * b_last, smem + 16u * b_last, 0u, hi & 15u);
                body_hi = 16u * b_last;
            }
            if (body_hi > body_lo)
                bulk_s2g(g + body_lo, smem + body_lo, body_hi - body_lo);
        }
    }
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");       /* the image must outlive the engine's reads */
}

/* generic (global-memory) tiles of a job: the CTA has just composed bytes [gbase, gbase + total) into its own
   buffer; after a barrier it copies that range to the peers (16-byte blocks where whole, bytes at the ends) */
__device__ __forceinline__ void copy_range_to_peers(const uint8_t *gown, uint8_t *const *s_pb, uint32_t npeers, uint64_t gbase,
    uint32_t total)
{
    const uint64_t end = gbase + total;
    uint64_t body_lo = (gbase + 15ull) & ~15ull, body_hi = end & ~15ull;
    if (body_hi <= body_lo)
        body_lo = body_hi = end;
    for (uint64_t b = body_lo + 16ull * threadIdx.x; b < body_hi; b += 16ull * TILE) {
        const uint4 v = *reinterpret_cast<const uint4 *>(gown + b);
        for (uint32_t q = 0; q < npeers; q++)
            stg_v4(s_pb[q] + b, v);
    }
    for (uint64_t i = gbase + threadIdx.x; i < body_lo; i += TILE)
        for (uint32_t q = 0; q < npeers; q++)
            s_pb[q][i] = gown[i];
    for (uint64_t i = body_hi + threadIdx.x; i < end; i += TILE)
        for (uint32_t q = 0; q < npeers; q++)
            s_pb[q][i] = gown[i];
}

/* Block-wide exclusive scan of one value per thread (two barriers). */
template <typename T>
__device__ __forceinline__ T block_scan(T *warp_sum /* smem[WARPS] */, T v, T *total)
{
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    T incl = v;
    #pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        T up = __shfl_up_sync(0xFFFFFFFFu, incl, d);
        if (lane >= (uint32_t)d)
            incl += up;
    }
    __syncthreads();                            /* warp_sum may still be read from a previous use */
    if (lane == 31)
        warp_sum[warp] = incl;
    __syncthreads();
    T before = 0, tot = 0;
    #pragma unroll
    for (int w = 0; w < WARPS; w++) {
        T s = warp_sum[w];
        if ((uint32_t)w < warp)
            before += s;
        tot += s;
    }
    *total = tot;
    return before + incl - v;
}

/*
 * ---- L2 lookahead ----
 * Every compose CTA starts with a chain of dependent round trips: its records' offsets and metadata, then the
 * bytes they point at.  So the CTA of tile k also asks the memory system to bring the first link of that chain for
 * tile k + D into L2 (cp.async.bulk.prefetch.L2, SASS UBLKPF): the tile's slices of the per-record arrays
 * (offsets, type ids, ttls, port flags), at addresses known from the tile index alone.  The payload kernel also
 * prefetches the second link, its address bytes and port values, between two offsets its lanes load at CTA start;
 * those offsets are not validated yet, so a reversed or oversized range is dropped and every range is clipped to
 * the caller's buffer.  D is half a wave of the launch (PathParams / JsonParams::lookahead, from the host's
 * occupancy figure; 0 = off): tile k + D starts about half a CTA lifetime later, when the prefetch has landed.  The
 * lanes of the last warp issue it, one array per lane, off the tile's own chain (thread 0, warp 0).
 *
 * Measured on an H100 (DESIGN.md §4): prefetching the path kernel's byte ranges (domains, hostnames, which its bulk
 * copies fetch anyway) made the step slower at every distance from a quarter of a wave to two waves.
 */
__device__ __forceinline__ void prefetch_l2(const void *base, uint64_t lo, uint64_t hi, uint64_t limit)
{
    hi = min(hi, limit);
    const uintptr_t a = ((uintptr_t)base + lo + 15u) & ~(uintptr_t)15, b = ((uintptr_t)base + hi) & ~(uintptr_t)15;
    if (base && hi > lo && b > a)
        asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(a), "r"((uint32_t)(b - a)));
}

/* elements [r0, r1) of an array of n elements of `esz` bytes (NULL: absent) */
__device__ __forceinline__ void prefetch_slice(const void *a, uint32_t esz, uint64_t r0, uint64_t r1, uint64_t n)
{
    prefetch_l2(a, esz * r0, esz * r1, esz * n);
}

/* records [r0, r1) of the tile `lookahead` tiles after this CTA's (the caller has checked that it exists) */
__device__ __forceinline__ void look_tile(uint32_t lookahead, uint64_t n, uint64_t &r0, uint64_t &r1)
{
    r0 = ((uint64_t)blockIdx.x + lookahead) * TILE;
    r1 = min(r0 + TILE, n);
}

/*
 * ---- per-CTA phase stamps (development build only: -DREGK_PHASE_STAMPS, tools/tile_phases.py) ----
 * Thread 0 of every compose CTA stores clock64() at five points of its tile, and the SM it ran on, into
 * g_phase_buf[kernel][tile][8] (kernel 0: paths, 1: payloads; set by regk_phase_stamps()).
 */
#ifdef REGK_PHASE_STAMPS
__device__ unsigned long long *g_phase_buf;
__device__ unsigned long long g_phase_cap;
__device__ __forceinline__ void phase_stamp(uint32_t kernel, uint32_t phase)
{
    if (threadIdx.x == 0 && g_phase_buf && blockIdx.x < g_phase_cap) {
        unsigned long long *e = g_phase_buf + ((unsigned long long)kernel * g_phase_cap + blockIdx.x) * 8u;
        e[phase] = clock64();
        if (phase == 0) {
            uint32_t sm;
            asm volatile("mov.u32 %0, %%smid;" : "=r"(sm));
            e[7] = sm;
        }
    }
}
#define REGK_PHASE(kernel, phase) phase_stamp(kernel, phase)
#else
#define REGK_PHASE(kernel, phase) ((void)0)
#endif

/*
 * Two-level totals instead of a scan pass: producers add each warp's byte count into tile_total[tile]
 * (u32) and super_total[tile / SUPER] (u64) with atomics; a consumer CTA derives its own exclusive base
 * as  sum(super_total[0 .. tile/SUPER)) + sum(tile_total[SUPER*(tile/SUPER) .. tile))  — at most
 * ntiles/SUPER + SUPER - 1 loads, done by warp 0 while the other warps load their records' metadata.
 * Kernel boundaries are the only synchronisation.  (Tried and dropped, with measurements in DESIGN.md:
 * a chained look-back scan, a fence + last-CTA scan, a separate single-CTA scan kernel.)
 */
constexpr uint32_t SUPER = 64;

__device__ __forceinline__ void add_tile_total(uint32_t *tile_total, unsigned long long *super_total, uint32_t tile,
    uint32_t warp_bytes)
{
    if (warp_bytes) {
        atomicAdd(tile_total + tile, warp_bytes);
        atomicAdd(super_total + tile / SUPER, (unsigned long long)warp_bytes);
    }
}

/* call from warp 0 (all 32 lanes); every lane returns the tile's exclusive base */
__device__ __forceinline__ unsigned long long tile_base_from_totals(const uint32_t *tile_total,
    const unsigned long long *super_total, uint32_t tile)
{
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t nsuper = tile / SUPER;
    unsigned long long acc = 0;
    for (uint32_t i = lane; i < nsuper; i += 32)
        acc += super_total[i];
    for (uint32_t i = nsuper * SUPER + lane; i < tile; i += 32)
        acc += tile_total[i];
    #pragma unroll
    for (int d = 16; d > 0; d >>= 1)
        acc += __shfl_xor_sync(0xFFFFFFFFu, acc, d);
    return acc;
}

__device__ __forceinline__ void report_bad(DevStatus *st, uint32_t bad, uint64_t rec)
{
    if (bad) {
        atomicOr(&st->bad_bits, bad);
        atomicMax(&st->first_bad, ~(unsigned long long)rec);   /* zero-initialised: max of ~rec == min rec */
    }
}

/* ======================================================= payload metadata == */

struct JsonParams {
    uint64_t n;
    const uint8_t *type_id;
    const uint8_t *addr_bytes;
    const uint32_t *addr_off;
    const int32_t *ttl;                 /* NULL: no record has a ttl */
    const uint32_t *ports_off;          /* NULL: no record has ports */
    const uint32_t *ports;
    const uint8_t *ports_present;       /* NULL: present iff k > 0 */
    const uint8_t *frag_blob;           /* TypeFrag[ntypes] followed by fragment bytes (word aligned) */
    uint32_t ntypes;
    uint32_t blob_bytes;                /* multiple of 16 */
    uint8_t *out_bytes;
    unsigned long long *out_off;
    uint64_t out_capacity;
    uint64_t rec0;                      /* index of this chunk's first record in the caller's batch (error reports) */
    const unsigned long long *base_in;  /* optional: payload bytes of all earlier chunks (host pipelining) */
    unsigned long long *base_out;       /* optional: *base_in + this chunk's payload bytes */
    uint32_t *tile_total;               /* [ntiles] payload bytes per tile, accumulated by the producer kernel */
    unsigned long long *super_total;    /* [ntiles / SUPER + 1] */
    DevStatus *status;
    uint64_t addr_limit, ports_limit;   /* bytes behind addr_bytes / elements behind ports (trusted) */
    uint32_t out_cap;                   /* shared-memory budget of the output image */
    uint32_t force_generic;
    uint32_t lookahead;                 /* tiles between a CTA and the tile whose inputs it prefetches (0: none) */
    PeerDst peer;                       /* multi-GPU job: the other ranks' whole-job payload buffers */
};

/* everything the payload of record r depends on except the address bytes */
struct JsonMeta {
    uint32_t tid, a0, al, p0, k;
    int32_t ttl;
    bool has_ttl, has_ports;
    uint32_t bad;
};

__device__ __forceinline__ JsonMeta json_meta(const JsonParams &p, uint64_t r)
{
    JsonMeta m;
    m.bad = 0;
    m.tid = p.type_id[r];
    if (m.tid >= p.ntypes) {
        m.bad |= BAD_TYPE_ID;
        m.tid = 0;
    }
    m.a0 = p.addr_off[r];
    uint32_t a1 = p.addr_off[r + 1];
    if (a1 < m.a0 || a1 > p.addr_limit) {
        m.bad |= BAD_TOO_LARGE;
        a1 = m.a0 = 0;
    }
    m.al = a1 - m.a0;
    if (m.al == 0)
        m.bad |= BAD_ADDR_BYTE;         /* a falsy adminIp means "auto-detect" upstream (register.js:143) */
    m.ttl = p.ttl ? p.ttl[r] : INT32_MIN;
    m.has_ttl = m.ttl != INT32_MIN;
    m.p0 = 0;
    m.k = 0;
    if (p.ports_off) {
        m.p0 = p.ports_off[r];
        uint32_t p1 = p.ports_off[r + 1];
        if (p1 < m.p0 || p1 > p.ports_limit) {
            m.bad |= BAD_TOO_LARGE;
            p1 = m.p0 = 0;
        }
        m.k = p1 - m.p0;
    }
    m.has_ports = p.ports_present ? (p.ports_present[r] != 0) : (m.k > 0);
    if (!m.has_ports)
        m.k = 0;
    return m;
}

__device__ __forceinline__ uint32_t json_meta_len(const JsonParams &p, const JsonMeta &m, const TypeFrag &tf)
{
    /* up to four port values by predicated loads issued together (SRV records rarely carry more), then a loop */
    const uint32_t *pp = p.ports + m.p0;
    const uint32_t k = m.k;
    uint32_t port_digits = 0;
    if (k) {                                                /* skipped by warps whose records carry no ports */
        const uint32_t v0 = pp[0], v1 = k > 1u ? pp[1] : 0u, v2 = k > 2u ? pp[2] : 0u, v3 = k > 3u ? pp[3] : 0u;
        port_digits = ndigits_u32(v0) + (k > 1u ? ndigits_u32(v1) : 0u) + (k > 2u ? ndigits_u32(v2) : 0u) +
                      (k > 3u ? ndigits_u32(v3) : 0u);
        for (uint32_t i = 4; i < k; i++)
            port_digits += ndigits_u32(pp[i]);
    }
    return json_length(tf.f1_len, tf.f2_len, m.al, m.has_ttl, m.ttl, m.has_ports, m.k, port_digits);
}

/* lookahead, payload metadata of records [r0, r1): lane j < 5 takes one array */
__device__ __forceinline__ void look_json(const JsonParams &p, uint32_t j, uint64_t r0, uint64_t r1)
{
    if (j == 0)
        prefetch_slice(p.type_id, 1, r0, r1, p.n);
    else if (j == 1)
        prefetch_slice(p.addr_off, 4, r0, r1 + 1, p.n + 1);
    else if (j == 2)
        prefetch_slice(p.ttl, 4, r0, r1, p.n);
    else if (j == 3)
        prefetch_slice(p.ports_off, 4, r0, r1 + 1, p.n + 1);
    else if (j == 4)
        prefetch_slice(p.ports_present, 1, r0, r1, p.n);
}

/* lookahead, payload kernel only: the second link of its chain, the address bytes (lane 5) and port values (lane 6),
   lie between two entries of the offsets array returned here; the lane loads them at CTA start */
__device__ __forceinline__ const uint32_t *look_json_bounds(const JsonParams &p, uint32_t j)
{
    return j == 5 ? p.addr_off : j == 6 ? p.ports_off : nullptr;
}

/* b0, b1: the two offsets look_json_bounds named, not validated yet: a reversed range, or one larger than four image
   budgets, is dropped; the rest is clipped to the buffer */
__device__ __forceinline__ void look_json_bytes(const JsonParams &p, uint32_t j, uint32_t b0, uint32_t b1)
{
    if (b1 < b0 || b1 - b0 > 4u * p.out_cap)
        return;
    if (j == 5)
        prefetch_l2(p.addr_bytes, b0, b1, p.addr_limit);
    else if (j == 6)
        prefetch_l2(p.ports, 4ull * b0, 4ull * b1, 4ull * p.ports_limit);
}

/* ================================================================ paths == */

struct PathParams {
    uint64_t n;
    const uint8_t *domain_bytes;
    const uint32_t *domain_off;
    const uint8_t *host_bytes;
    const uint32_t *host_off;           /* NULL: fixed stride */
    uint32_t host_stride;
    uint8_t *out_bytes;
    unsigned long long *out_off;        /* [n+1] */
    uint64_t out_capacity;
    uint64_t rec0;                      /* index of this chunk's first record in the caller's batch (error reports) */
    uint64_t off_bias;                  /* added to every output offset: a chunk of a larger batch keeps absolute
                                           input offsets but numbers its records from 0 (host pipelining) */
    uint32_t exact;                     /* 0: closed-form offsets; 1: bases from tile_total / super_total */
    uint32_t *tile_total;               /* [ntiles]   exact path bytes per tile (regk_path_len_kernel) */
    unsigned long long *super_total;    /* [ntiles / SUPER + 1] */
    DevStatus *status;
    uint64_t dom_limit, host_limit;     /* bytes behind domain_bytes / host_bytes (trusted, from the caller) */
    uint32_t dom_cap, host_cap, out_cap;        /* shared-memory budgets in bytes */
    uint32_t force_generic;
    uint32_t lookahead;                 /* tiles between a CTA and the tile whose inputs it prefetches (0: none) */
    const unsigned long long *bias_in;  /* optional, device: added to off_bias (job: path bytes of the ranks before this one) */
    PeerDst peer;                       /* multi-GPU job: the other ranks' whole-job path buffers */
};

/* lookahead of the path kernel, records [r0, r1): lanes 0-1 take the path offsets, lanes 2-6 the side job's payload
   metadata */
template <bool ALIAS>
__device__ __forceinline__ void look_path(const PathParams &p, const JsonParams &jp, bool side, uint32_t lane, uint64_t r0,
    uint64_t r1)
{
    if (lane == 0)
        prefetch_slice(p.domain_off, 4, r0, r1 + 1, p.n + 1);
    else if (!ALIAS && lane == 1)
        prefetch_slice(p.host_off, 4, r0, r1 + 1, p.n + 1);
    else if (side && lane >= 2)
        look_json(jp, lane - 2, r0, r1);
}

/* closed-form offset of record r's path when no label is empty: path_len = L + 2 + H (alias: L + 1) */
template <bool ALIAS>
__device__ __forceinline__ unsigned long long path_cf(const PathParams &p, uint64_t r)
{
    unsigned long long v = (unsigned long long)p.domain_off[r];
    if (ALIAS)
        return v + r;
    return v + 2ull * r + (p.host_off ? (unsigned long long)p.host_off[r] : r * (unsigned long long)p.host_stride);
}

/*
 * Exact path lengths -> per-tile totals -> per-tile bases.  Only launched when the compose
 * kernel reported `needs_exact` (some domain has empty labels, which path.join drops).
 */
template <bool ALIAS>
__global__ void __launch_bounds__(TILE) regk_path_len_kernel(const PathParams p)
{
    const uint32_t tile = blockIdx.x, t = threadIdx.x;
    const uint64_t r0 = (uint64_t)tile * TILE;
    const uint32_t nrec = (uint32_t)min((uint64_t)TILE, p.n - r0);
    uint32_t len = 0;
    if (t < nrec) {
        const uint64_t r = r0 + t;
        const uint32_t d0 = p.domain_off[r], d1 = p.domain_off[r + 1];
        const uint32_t L = (d1 >= d0 && d1 <= p.dom_limit) ? d1 - d0 : 0;   /* corrupt offsets: flagged by the compose kernel */
        uint32_t H = 0;
        if (!ALIAS) {
            if (p.host_off) {
                const uint32_t a = p.host_off[r], b = p.host_off[r + 1];
                H = b >= a ? b - a : 0;
            } else {
                H = p.host_stride;
            }
        }
        const GuardedWords dsrc{reinterpret_cast<const uint32_t *>(p.domain_bytes)};
        len = path_length(scan_domain(dsrc, d0, L), L, H, ALIAS);
    }
    #pragma unroll
    for (int d = 16; d > 0; d >>= 1)
        len += __shfl_xor_sync(0xFFFFFFFFu, len, d);
    if ((t & 31u) == 0)
        add_tile_total(p.tile_total, p.super_total, tile, len);
}

/* payload lengths of this tile -> tile_total / super_total (consumed by regk_json_kernel) */
__device__ __forceinline__ void payload_length_side_job(const JsonParams &jp, const JsonMeta &jm, const TypeFrag &jtf,
    bool live, uint32_t tile)
{
    uint32_t jl = live ? json_meta_len(jp, jm, jtf) : 0;
    #pragma unroll
    for (int d = 16; d > 0; d >>= 1)
        jl += __shfl_xor_sync(0xFFFFFFFFu, jl, d);
    if ((threadIdx.x & 31u) == 0)
        add_tile_total(jp.tile_total, jp.super_total, tile, jl);
}

/*
 * regk_path_kernel: one CTA per tile of TILE records.
 *  - tile inputs (contiguous byte ranges of domain_bytes / host_bytes) are staged into shared memory by two
 *    cp.async.bulk copies (TMA engine) issued by one thread, completion on an mbarrier — no per-thread
 *    staging instructions;
 *  - `jp.n != 0` turns on a side job: the kernel also computes the PAYLOAD length of each of its records
 *    (metadata only; those loads overlap the staging) and adds the per-warp sums into jp.tile_total /
 *    jp.super_total, from which every CTA of regk_json_kernel derives its base — no separate pass over the
 *    payload metadata and no scan launch.
 */
/* CTA-uniform facts about a tile, worked out once by thread 0 and read by everybody after one barrier */
struct TilePlan {
    unsigned long long tile_base;       /* where the tile's output starts in the packed stream */
    unsigned long long HB0;             /* start of the tile's hostnames in host_bytes */
    uint32_t D0, D1, HA1;               /* tile extents (HA1: end of the hostnames, variable-length case) */
    uint32_t nd, nh;                    /* bytes staged for domains / hostnames (multiples of 16) */
    uint32_t host_span;                 /* bytes of this tile's hostnames */
    uint32_t tile_total;
    uint32_t flags;                     /* PLAN_* */
};
enum : uint32_t { PLAN_BROKEN = 1, PLAN_FITS = 2, PLAN_BULK = 4, PLAN_ROOM = 8 };

template <bool ALIAS, bool EXACT>
__global__ void __launch_bounds__(TILE, REGK_MINB_PATH) regk_path_kernel(const PathParams p, const JsonParams jp)
{
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ uint32_t warp_sum[WARPS];
    __shared__ __align__(8) uint64_t s_bar;
    __shared__ TilePlan s_plan;
    __shared__ uint8_t *s_pb[REGK_MAX_PEERS - 1];
    __shared__ unsigned long long *s_po[REGK_MAX_PEERS - 1];
    REGK_PHASE(0, 0);
    const uint32_t npeers = p.peer.n;
    if (npeers)
        peer_tables(p.peer, s_pb, s_po);                        /* published by the plan barrier */
    uint8_t *s_dom = smem + 16;                                 /* staged domain bytes (16 bytes of front padding):
                                                                   lower-cased, '.' -> '/' */
    uint8_t *s_bits = s_dom + p.dom_cap + 32;                   /* 1 bit per staged domain byte: was '.' */
    uint8_t *s_host = s_bits + p.dom_cap / 8 + 16;
    uint8_t *s_out = s_host + (ALIAS ? 0 : p.host_cap + 32);

    const uint32_t tile = blockIdx.x;
    const uint32_t t = threadIdx.x;
    const uint64_t r0 = (uint64_t)tile * TILE;
    const uint32_t nrec = (uint32_t)min((uint64_t)TILE, p.n - r0);
    const bool live = t < nrec;
    const uint32_t tl = live ? t : 0u;                          /* idle threads shadow record 0 of the tile */
    const uint64_t r = r0 + tl;
    constexpr bool exact = EXACT;               /* compile-time: the closed-form kernel carries none of the redo's code */
    const bool var_host = !ALIAS && p.host_off != nullptr;
    const uint32_t per_rec = ALIAS ? 1u : 2u;                   /* '/' per record, plus '/' before the hostname */

    /* ---- thread 0: plan the tile, start the bulk copies ---- */
    if (t == 0) {
        mbar_init(&s_bar, 1);
        TilePlan q;
        q.D0 = p.domain_off[r0];
        q.D1 = p.domain_off[r0 + nrec];
        unsigned long long HB1 = 0;
        q.HB0 = 0;
        q.HA1 = 0;
        if (var_host) {
            q.HB0 = p.host_off[r0];
            q.HA1 = p.host_off[r0 + nrec];
            HB1 = q.HA1;
        } else if (!ALIAS) {
            q.HB0 = r0 * p.host_stride;
            HB1 = q.HB0 + (unsigned long long)nrec * p.host_stride;
        }
        const bool broken = q.D1 < q.D0 || q.D1 > p.dom_limit || (!ALIAS && (HB1 < q.HB0 || HB1 > p.host_limit));
        const uint32_t dom_span = q.D1 - q.D0, host_span = (uint32_t)(HB1 - q.HB0);
        const uint32_t dom_lead = q.D0 & 15u, host_lead = (uint32_t)q.HB0 & 15u;
        q.nd = (dom_lead + dom_span + 15u) & ~15u;
        q.nh = ALIAS ? 0u : (host_lead + host_span + 15u) & ~15u;
        const bool fits = !broken && !p.force_generic && dom_lead + dom_span <= p.dom_cap &&
            (ALIAS || host_lead + host_span <= p.host_cap) && dom_span + host_span + 2u * nrec + 16u <= p.out_cap;
        /* whole 16-byte blocks must stay inside the caller's buffers for the bulk copies */
        const bool bulk = fits && (unsigned long long)(q.D0 & ~15u) + q.nd <= p.dom_limit &&
            (ALIAS || (q.HB0 & ~15ull) + q.nh <= p.host_limit);
        if (bulk) {
            mbar_expect_tx(&s_bar, q.nd + q.nh);
            if (q.nd)
                bulk_g2s(s_dom, p.domain_bytes + (q.D0 & ~15u), q.nd, &s_bar);
            if (q.nh)
                bulk_g2s(s_host, p.host_bytes + (q.HB0 & ~15ull), q.nh, &s_bar);
        }
        /* closed-form placement: slot = L + 2 + H bytes per record (alias: L + 1) */
        q.tile_base = (unsigned long long)q.D0 + q.HB0 + (unsigned long long)per_rec * r0 + p.off_bias +
            (p.bias_in ? *p.bias_in : 0ull);
        q.tile_total = dom_span + host_span + per_rec * nrec;
        q.host_span = host_span;
        q.flags = (broken ? PLAN_BROKEN : 0u) | (fits ? PLAN_FITS : 0u) | (bulk ? PLAN_BULK : 0u);
        if (!exact && !broken && q.tile_base + q.tile_total <= p.out_capacity)
            q.flags |= PLAN_ROOM;
        s_plan = q;
    }

    /* ---- everybody: this record's offsets; the side job's metadata loads overlap the staging ---- */
    const uint32_t d0 = p.domain_off[r], d1 = p.domain_off[r + 1];
    uint32_t ha = 0, hb = 0;
    if (var_host) {
        ha = p.host_off[r];
        hb = p.host_off[r + 1];
    }
    const bool side = !EXACT && jp.n != 0;
    JsonMeta jm;
    TypeFrag jtf;
    if (side) {
        jm = json_meta(jp, r);
        jtf = reinterpret_cast<const TypeFrag *>(jp.frag_blob)[jm.tid];
    }
    unsigned long long exact_base = 0;
    if (exact && t < 32)
        exact_base = tile_base_from_totals(p.tile_total, p.super_total, tile);
    if (exact && t == 0)
        *reinterpret_cast<unsigned long long *>(warp_sum) = exact_base;     /* read back after the barrier, before any scan */
    if (p.lookahead && tile + p.lookahead < gridDim.x && t >= TILE - 32) {
        uint64_t l0, l1;
        look_tile(p.lookahead, p.n, l0, l1);
        look_path<ALIAS>(p, jp, side, t & 31u, l0, l1);
    }
    __syncthreads();                                            /* plan, mbarrier init (and exact base) published */
    REGK_PHASE(0, 1);

    /* the side job runs while the bulk copies are in flight: its second-hop loads (port values) cost nothing
       here, and its registers are free again before the composing starts */
    if (side)
        payload_length_side_job(jp, jm, jtf, live, tile);

    const uint32_t flags = s_plan.flags;
    const uint32_t D0 = s_plan.D0;
    unsigned long long tile_base = s_plan.tile_base;
    uint32_t tile_total = s_plan.tile_total;
    bool room = flags & PLAN_ROOM;
    if (exact) {
        tile_base = *reinterpret_cast<const unsigned long long *>(warp_sum) + p.off_bias + (p.bias_in ? *p.bias_in : 0ull);
        tile_total = p.tile_total[tile];
        room = !(flags & PLAN_BROKEN) && tile_base + tile_total <= p.out_capacity;
        __syncthreads();                                        /* warp_sum is about to be reused by block_scan */
    }
    uint32_t bad = 0;
    /* a record whose own offsets are inconsistent is emptied and reported; the tile carries on */
    bool rec_ok = d1 >= d0 && d0 >= D0 && d1 <= s_plan.D1;
    uint32_t hrel, H;
    if (ALIAS) {
        hrel = 0;
        H = 0;
    } else if (var_host) {
        rec_ok = rec_ok && hb >= ha && ha >= (uint32_t)s_plan.HB0 && hb <= s_plan.HA1;
        hrel = ha - (uint32_t)s_plan.HB0;
        H = hb - ha;
    } else {
        hrel = tl * p.host_stride;
        H = p.host_stride;
    }
    uint32_t L = d1 - d0;
    if (!live || !rec_ok) {
        L = 0;
        H = 0;
    }
    if (live && (!rec_ok || (flags & PLAN_BROKEN)))
        bad = BAD_TOO_LARGE;
    uint32_t local = rec_ok ? (d0 - D0) + hrel + per_rec * tl : 0u;
    const uint32_t slot = L + H + per_rec;

    if (flags & PLAN_BROKEN) {
        /* tile extents outside the buffers: nothing is read or written */
    } else if (flags & PLAN_FITS) {
        const uint32_t nd = s_plan.nd, nh = s_plan.nh;
        if (flags & PLAN_BULK) {
            mbar_wait(&s_bar, 0);
        } else {                                                /* the stream's last blocks */
            stage_in(s_dom, p.domain_bytes, D0, s_plan.D1, p.dom_limit);
            if (!ALIAS)
                stage_in(s_host, p.host_bytes, s_plan.HB0, s_plan.HB0 + s_plan.host_span, p.host_limit);
            __syncthreads();
        }
        REGK_PHASE(0, 2);
        /* cooperative pre-pass: lower-case, dot bitmap, '.' -> '/', fence (vectorised, no divergence) */
        uint32_t *dom_w = reinterpret_cast<uint32_t *>(s_dom);
        const uint32_t *bits_w = reinterpret_cast<const uint32_t *>(s_bits);
        const uint32_t *host_w = reinterpret_cast<const uint32_t *>(s_host);
        uint32_t suspicious = prepass_domain(dom_w, reinterpret_cast<uint16_t *>(s_bits), nd >> 4, t, TILE);
        if (!ALIAS)
            suspicious |= prepass_host(host_w, nh >> 4, t, TILE);
        suspicious = __syncthreads_or(suspicious != 0);
        const uint32_t doff = (D0 & 15u) + (d0 - D0);
        const uint32_t hoff = ((uint32_t)s_plan.HB0 & 15u) + hrel;
        const DomainInfo di = domain_info(bits_w, rec_ok ? doff : 0u, L);
        if (suspicious) {
            /* something in or next to this tile is outside the fence: find out exactly which records */
            bad |= recheck_domain(s_dom, bits_w, doff, L);
            if (!ALIAS && live && rec_ok)
                bad |= check_host(PaddedWords{host_w}, hoff, H);
        } else if (!ALIAS && live && rec_ok && H <= 2) {
            bad |= check_host(PaddedWords{host_w}, hoff, H);    /* "", "." and ".." have no bad byte */
        }
        const uint32_t len = (live && rec_ok) ? path_length2(di, L, H, ALIAS) : 0;
        if (exact) {
            uint32_t tot;
            local = block_scan<uint32_t>(warp_sum, len, &tot);
        } else if (live && len != slot) {
            atomicOr(&p.status->needs_exact, 1u);               /* empty labels: redo with exact offsets */
        }
        if (live) {
            p.out_off[r] = tile_base + local;
            for (uint32_t q = 0; q < npeers; q++)
                s_po[q][r] = tile_base + local;
        }
        if (room) {
            WordSink sink;
            sink.init(reinterpret_cast<uint32_t *>(s_out), local + ((uint32_t)tile_base & 15u));
            if (live && rec_ok) {
                if (!ALIAS && H >= 24u)                          /* a long hostname follows: label blocks may overshoot */
                    emit_path2<ALIAS, true>(dom_w, bits_w, doff, L, di, host_w, hoff, H, sink);
                else
                    emit_path2<ALIAS, false>(dom_w, bits_w, doff, L, di, host_w, hoff, H, sink);
            }
            __syncthreads();
            if (live)
                sink.tail();                                    /* phase B: shared boundary words */
            fence_proxy_async();
            __syncthreads();
            REGK_PHASE(0, 3);
            if (npeers)
                flush_out_job(p.out_bytes, s_pb, npeers, s_out, tile_base, tile_total);
            else
                flush_out(p.out_bytes, s_out, tile_base, tile_total);
            REGK_PHASE(0, 4);
        }
    } else {
        /* generic path: compose straight from / to global memory */
        if (t == 0)
            atomicAdd(&p.status->generic_tiles, 1u);
        const unsigned long long HB0 = s_plan.HB0;
        const GuardedWords dsrc{reinterpret_cast<const uint32_t *>(p.domain_bytes)};
        const GuardedWords hsrc{reinterpret_cast<const uint32_t *>(p.host_bytes + (var_host ? 0 : HB0))};
        const uint32_t hoff = var_host ? (uint32_t)HB0 + hrel : hrel;
        const DomainStats st = scan_domain(dsrc, d0, L);
        bad |= st.bad;
        if (!ALIAS && live && rec_ok)
            bad |= check_host(hsrc, hoff, H);
        const uint32_t len = (live && rec_ok) ? path_length(st, L, H, ALIAS) : 0;
        if (exact) {
            uint32_t tot;
            local = block_scan<uint32_t>(warp_sum, len, &tot);
        } else if (live && len != slot) {
            atomicOr(&p.status->needs_exact, 1u);
        }
        if (live) {
            p.out_off[r] = tile_base + local;
            for (uint32_t q = 0; q < npeers; q++)
                s_po[q][r] = tile_base + local;
        }
        if (room && live && rec_ok) {
            ByteSink sink;
            sink.init(p.out_bytes + tile_base + local);
            emit_path<ALIAS>(dsrc, d0, L, hsrc, hoff, H, sink);
        }
        if (npeers && room) {                                   /* CTA-uniform */
            __syncthreads();
            copy_range_to_peers(p.out_bytes, s_pb, npeers, tile_base, tile_total);
        }
    }
    if (!room && !(flags & PLAN_BROKEN) && t == 0)
        atomicOr(&p.status->overflow, 1u);
    if (live)
        report_bad(p.status, bad, p.rec0 + r);
    if (r0 + nrec == p.n && t == 0) {
        if (p.peer.job) {
            /* job: the entry after the shard's last record belongs to the next rank (or is the job's closing
               entry, written by the exchange kernel); report the shard's own byte count */
            p.status->path_total = tile_base + tile_total - (p.bias_in ? *p.bias_in : 0ull) - p.off_bias;
        } else {
            p.out_off[p.n] = tile_base + tile_total;
            p.status->path_total = tile_base + tile_total;
        }
    }
}

/* ============================================================= payloads == */

/*
 * Payload lengths from the metadata only (no string bytes) -> per-tile totals -> per-tile bases.
 * Only used when the path half is skipped (REGK_NO_PATH).  Persistent grid: each CTA walks tiles
 * blockIdx.x, +gridDim.x, ...; a warp sums its 32 records with shuffles and adds the sum to the tile's
 * totals (zeroed by the host) with atomics.
 */
__global__ void __launch_bounds__(TILE) regk_json_len_kernel(const JsonParams p, uint32_t ntiles)
{
    const uint32_t t = threadIdx.x, lane = t & 31u;
    for (uint32_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const uint64_t r = (uint64_t)tile * TILE + t;
        uint32_t len = 0;
        if (r < p.n) {
            const JsonMeta m = json_meta(p, r);
            const TypeFrag tf = reinterpret_cast<const TypeFrag *>(p.frag_blob)[m.tid];
            len = json_meta_len(p, m, tf);
        }
        #pragma unroll
        for (int d = 16; d > 0; d >>= 1)
            len += __shfl_xor_sync(0xFFFFFFFFu, len, d);
        if (lane == 0)
            add_tile_total(p.tile_total, p.super_total, tile, len);
    }
}

/* CTA-uniform facts of a payload tile, worked out by warp 0 */
struct JsonPlan {
    unsigned long long tile_base;
    uint32_t tile_total;
    uint32_t flags;                     /* PLAN_ROOM | PLAN_FITS */
};

__global__ void __launch_bounds__(TILE, REGK_MINB_JSON) regk_json_kernel(const JsonParams p)
{
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ uint32_t warp_sum[WARPS];
    __shared__ __align__(8) uint64_t s_bar;
    __shared__ JsonPlan s_plan;
    __shared__ uint8_t *s_pb[REGK_MAX_PEERS - 1];
    __shared__ unsigned long long *s_po[REGK_MAX_PEERS - 1];
    REGK_PHASE(1, 0);
    const uint32_t npeers = p.peer.n;
    if (npeers)
        peer_tables(p.peer, s_pb, s_po);                        /* published by the scan's barriers */
    uint8_t *s_blob = smem;
    uint8_t *s_out = smem + p.blob_bytes;

    const uint32_t t = threadIdx.x;
    const uint32_t tile = blockIdx.x;
    const uint64_t r0 = (uint64_t)tile * TILE;
    const uint32_t nrec = (uint32_t)min((uint64_t)TILE, p.n - r0);
    const bool live = t < nrec;
    const uint64_t r = r0 + (live ? t : 0);

    /* warp 0: fragment table by one bulk copy (TMA), this tile's base from the two-level totals */
    if (t < 32) {
        if (t == 0) {
            mbar_init(&s_bar, 1);
            mbar_expect_tx(&s_bar, p.blob_bytes);
            bulk_g2s(s_blob, p.frag_blob, p.blob_bytes, &s_bar);
        }
        const unsigned long long b = tile_base_from_totals(p.tile_total, p.super_total, tile) + (p.base_in ? *p.base_in : 0ull);
        if (t == 0) {
            JsonPlan q;
            q.tile_base = b;
            q.tile_total = p.tile_total[tile];
            q.flags = (b + q.tile_total <= p.out_capacity ? PLAN_ROOM : 0u) |
                (!p.force_generic && q.tile_total + 16u <= p.out_cap ? PLAN_FITS : 0u);
            s_plan = q;
        }
    }

    const bool look = p.lookahead && tile + p.lookahead < gridDim.x && t >= TILE - 32;
    uint32_t lb0 = 0, lb1 = 0;
    if (look) {
        uint64_t l0, l1;
        look_tile(p.lookahead, p.n, l0, l1);
        look_json(p, t & 31u, l0, l1);
        if (const uint32_t *bo = look_json_bounds(p, t & 31u)) {
            lb0 = bo[l0];
            lb1 = bo[l1];
        }
    }
    const JsonMeta m = json_meta(p, r);
    uint32_t bad = m.bad;
    const uint32_t a0 = m.a0, al = m.al, k = m.k;

    /* first 16 address bytes -> registers, fenced */
    const GuardedWords asrc{reinterpret_cast<const uint32_t *>(p.addr_bytes)};
    uint32_t aw[4] = {0, 0, 0, 0};
    {
        const uint32_t n16 = al < 16u ? al : 16u;
        const uint32_t sh = (a0 & 3u) * 8u;
        uint32_t wi = a0 >> 2;
        uint32_t lo = n16 ? asrc.word(wi) : 0u;
        #pragma unroll
        for (int w = 0; w < 4; w++) {
            if (n16 > 4u * w) {
                const uint32_t nb = min(4u, n16 - 4u * w);
                const uint32_t hi = asrc.word_hi(wi + 1, sh + 8u * nb > 32u || n16 > 4u * (w + 1));
                const uint32_t keep = low_bytes(nb);
                aw[w] = funnel_r(lo, hi, sh) & keep;
                if (addr_word_bad(aw[w], keep))
                    bad |= BAD_ADDR_BYTE;
                lo = hi;
                wi++;
            }
        }
        for (uint32_t i = a0 + 16u; i < a0 + al; i++) {     /* rare: address longer than 16 bytes */
            const uint32_t c = p.addr_bytes[i];
            if (c < 0x20u || c >= 0x80u || c == 0x22u || c == 0x5Cu)
                bad |= BAD_ADDR_BYTE;
        }
    }
    /* the record's length needs only its type's fragment lengths: read them from the global table (16 bytes, L2)
       so that nobody waits for warp 0's totals or the bulk copy before the scan; the scan's own barriers publish
       the plan and the mbarrier init */
    const TypeFrag tf = reinterpret_cast<const TypeFrag *>(p.frag_blob)[m.tid];
    const uint32_t len = live ? json_meta_len(p, m, tf) : 0;
    if (look)
        look_json_bytes(p, t & 31u, lb0, lb1);                 /* the bounds have landed by now */
    REGK_PHASE(1, 1);
    uint32_t tot;
    const uint32_t local = block_scan<uint32_t>(warp_sum, len, &tot);
    mbar_wait(&s_bar, 0);                                       /* fragment table has landed */
    REGK_PHASE(1, 2);
    const unsigned long long tile_base = s_plan.tile_base;
    const uint32_t tile_total = s_plan.tile_total;
    const uint32_t flags = s_plan.flags;
    if (live) {
        p.out_off[r] = tile_base + local;
        for (uint32_t q = 0; q < npeers; q++)
            s_po[q][r] = tile_base + local;
    }

    const PaddedWords blob{reinterpret_cast<const uint32_t *>(s_blob)};
    const uint32_t *ports = p.ports + m.p0;
    auto port = [ports](uint32_t i) { return ports[i]; };
    if (!(flags & PLAN_ROOM)) {
        if (t == 0)
            atomicOr(&p.status->overflow, 1u);
    } else if (flags & PLAN_FITS) {
        WordSink sink;
        sink.init(reinterpret_cast<uint32_t *>(s_out), local + ((uint32_t)tile_base & 15u));
        if (live)
            emit_json(blob, tf, aw, asrc, a0, al, m.has_ttl, m.ttl, m.has_ports, k, port, sink);
        __syncthreads();
        if (live)
            sink.tail();                                        /* phase B: shared boundary words */
        fence_proxy_async();
        __syncthreads();
        REGK_PHASE(1, 3);
        if (npeers)
            flush_out_job(p.out_bytes, s_pb, npeers, s_out, tile_base, tile_total);
        else
            flush_out(p.out_bytes, s_out, tile_base, tile_total);
        REGK_PHASE(1, 4);
    } else {
        if (t == 0)
            atomicAdd(&p.status->generic_tiles, 1u);
        if (live) {
            ByteSink sink;
            sink.init(p.out_bytes + tile_base + local);
            emit_json(blob, tf, aw, asrc, a0, al, m.has_ttl, m.ttl, m.has_ports, k, port, sink);
        }
        if (npeers) {                                           /* CTA-uniform */
            __syncthreads();
            copy_range_to_peers(p.out_bytes, s_pb, npeers, tile_base, tile_total);
        }
    }
    if (live)
        report_bad(p.status, bad, p.rec0 + r);
    if (r0 + nrec == p.n && t == 0) {
        if (p.peer.job) {
            p.status->json_total = tile_base + tile_total - (p.base_in ? *p.base_in : 0ull);    /* the shard's own bytes */
        } else {
            p.out_off[p.n] = tile_base + tile_total;
            p.status->json_total = tile_base + tile_total;
            if (p.base_out)
                *p.base_out = tile_base + tile_total;
        }
    }
}

}  /* namespace regk */
#endif /* REGK_KERNELS_CUH */
