/*
 * regk_api.cu — C-ABI (include/regk.h) over the sm_90a kernels.
 *
 * Host-side plumbing only: argument checks, device buffers, the per-type JSON
 * fragment table, launch configuration, status read-back.  All record bytes
 * are produced by the kernels in regk_kernels.cuh; there is no CPU
 * implementation of the path in this library.
 */
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/regk.h"
#include "regk_kernels.cuh"
#include "regk_gather.cuh"
#include "regk_peersync.cuh"
#include "regk_service.cuh"
#include "regk_jute.cuh"
#include "regk_decode.cuh"
#include "regk_parents.cuh"
#include "regk_skip.cuh"
#include "regk_mkdirp.cuh"
#include "regk_reconcile.cuh"
#include "regk_replies.cuh"
#include "regk_types.hpp"

using namespace regk;

namespace {

thread_local std::string g_create_error;

struct DevBuf {
    void *p = nullptr;
    size_t cap = 0;
};

struct HostBuf {
    void *p = nullptr;
    size_t cap = 0;
};

}  // namespace

struct regk_ctx {
    int device = 0;
    cudaStream_t own_stream = nullptr;
    cudaStream_t stream = nullptr;              /* the stream work is enqueued on */
    std::string err;
    int sm_count = 0;
    int max_smem_optin = 0;
    /* compose kernels' L2 lookahead: CTAs of one wave by dynamic shared memory (lookahead_tiles); index as in
       smem_attr_needs_raise (0 alias paths, 1 node paths, 2 payloads) */
    std::map<size_t, uint32_t> wave_ctas[3];

    /* type table */
    std::vector<std::string> types;             /* raw */
    std::vector<uint8_t> blob_host;             /* TypeFrag[] + fragments, padded to 16 */
    DevBuf blob_dev;
    uint32_t max_type_q = 0;                    /* longest escaped type */

    /* device staging of host batches */
    DevBuf in[11];
    /* outputs */
    DevBuf path_bytes, path_off, json_bytes, json_off, off32_p, off32_j;
    HostBuf h_path_bytes, h_path_off, h_json_bytes, h_json_off, h_running;
    cudaStream_t s_h2d = nullptr, s_d2h = nullptr;          /* host pipelining (run_pipelined, two-deep async) */
    /* "async" host batches alternate between two complete sets of staging, device outputs and pinned result
       buffers: batch k+1's H2D and kernels overlap batch k's D2H (issued when k+1 is submitted or k is
       finished, whichever comes first - the copy sizes are only known once k's kernels are done) */
    struct HostSet {
        DevBuf in[11];
        DevBuf path_bytes, path_off, json_bytes, json_off, off32_p, off32_j;
        HostBuf h_path_bytes, h_path_off, h_json_bytes, h_json_off;
        cudaEvent_t e_in = nullptr, e_out = nullptr;
    };
    HostSet hset[2];
    uint64_t hseq = 0;
    uint32_t *h_gather_flag = nullptr;          /* pinned: 1 = regk_gather_push found the whole-job buffers too small,
                                                   2 = a peer exchange of a job step timed out */
    /* multi-GPU job (regk_job_bind): description, exchange sequence number, per-slot bases {path base, path all,
       rec base, n all, payload base, payload all, -, -} on the device and their pinned host copies */
    double json_mean_seen = 0.0;                /* payload bytes per record of the batch finished last (same type table) ... */
    uint64_t json_est_seen = 0;                 /* ... and the a-priori estimate that batch had: the figure is reused only for
                                                   batches with the same estimate */
    bool json_learning = true;
    regk_job job{};
    bool job_bound = false;
    unsigned long long job_seq = 0;
    DevBuf job_bases;
    unsigned long long *h_job_bases = nullptr;
    /* device copy of the path stream of the batch finished last (regk_parent_dirs works on it) */
    const uint8_t *last_path_bytes = nullptr;
    const unsigned long long *last_path_off = nullptr;
    uint64_t last_n = 0;
    /* ... and of its payload stream (regk_jute_frames / regk_decode work on both) */
    const uint8_t *last_json_bytes = nullptr;
    const unsigned long long *last_json_off = nullptr;
    uint64_t last_json_n = 0;
    DevBuf jute_bytes, jute_off;
    HostBuf h_jute_bytes, h_jute_off;
    DevBuf dec_in[4], dec_rec, dec_dom, dec_ports;
    HostBuf h_dec_rec, h_dec_dom, h_dec_ports;
    const uint32_t *last_host_off = nullptr;
    uint32_t last_host_stride = 0;
    bool last_alias = false;
    DevBuf svc_in[7], svc_work;                 /* regk_service_records: staged inputs, status + tile totals */
    DevBuf par_len, par_slot, par_table, par_totals, par_unique;
    cudaEvent_t par_ev[2] = {nullptr, nullptr};
    HostBuf h_par_len, h_par_unique, h_par_count;
    /* regk_mkdirp_dirs (regk_mkdirp.cuh): its own parent pass, work lists, table, the set; regk_mkdirp_requests */
    enum { MK_PLEN, MK_PSLOT, MK_PTABLE, MK_PTOTALS, MK_PUNIQUE, MK_FLAGS, MK_LIST0, MK_LIST1, MK_TOTALS, MK_TABLE,
           MK_COUNT, MK_DREC, MK_DLEN, MK_DBYTES, MK_DOFF, MK_DEPTH, MK_INVALID, MK_ZERO, MK_FBYTES, MK_FOFF, MK_NBUF };
    DevBuf mk[MK_NBUF];
    HostBuf h_mk_count, h_mk_drec, h_mk_dlen, h_mk_dbytes, h_mk_doff, h_mk_depth, h_mk_invalid, h_mk_fbytes, h_mk_foff;
    cudaEvent_t mk_ev[4] = {nullptr, nullptr, nullptr, nullptr};
    bool mk_valid = false;                      /* the set of the last regk_mkdirp_dirs call is in mk[MK_D*] */
    uint64_t mk_n_dirs = 0, mk_bytes = 0;
    /* regk_reconcile / regk_reconcile_owned (regk_reconcile.cuh): staged snapshot and stats, tables, outputs, lists,
       versions, the gathered request streams; regk_reconcile_requests' frames */
    enum { RC_IN_PB, RC_IN_PO, RC_IN_JB, RC_IN_JO, RC_IN_VER, RC_IN_OWN, RC_TOBS, RC_TDES, RC_SLOTO, RC_HASHO, RC_SLOTD, RC_CLS,
           RC_MATCH, RC_OBSCLS, RC_TOTALS, RC_LIST0, RC_LEN0 = RC_LIST0 + RC_NLISTS, RC_VER0 = RC_LEN0 + RC_NGATHERS,
           RC_COUNT = RC_VER0 + RC_NVER, RC_GTOTALS, RC_G0B, RC_FBYTES = RC_G0B + 2 * RC_NGATHERS, RC_FOFF, RC_NBUF };
    DevBuf rc[RC_NBUF];
    HostBuf h_rc_count, h_rc_cls, h_rc_match, h_rc_obscls, h_rc_list[RC_NLISTS], h_rc_fbytes, h_rc_foff;
    cudaEvent_t rc_ev[2] = {nullptr, nullptr};
    bool rc_valid = false;                      /* the request streams of the last reconcile call are in rc[RC_G0B + 2 k] */
    bool rc_owned = false;                      /* ... and it was regk_reconcile_owned: versions in rc[RC_VER*] */
    uint32_t rc_zk_flags = 0;                   /* the CreateMode regk_reconcile_owned classified with */
    uint64_t rc_count[RC_NLISTS] = {};          /* create, update, dup, replace, delete */
    /* which batch finished last: bumped whenever the streams of the batch finished last change */
    uint64_t last_gen = 0;
    /* the last REGK_ZK_GETDATA framing: the batch it framed, xid_base, n (regk_read_replies reads its replies) */
    bool gd_valid = false;
    uint64_t gd_gen = 0, gd_n = 0;
    int32_t gd_xid = 0;
    /* regk_read_replies (regk_replies.cuh): staged stream, candidates, jump tables, per-record arrays, table, the nodes
       and the gathered snapshot */
    enum { RQ_STREAM, RQ_WORD, RQ_TOTALS, RQ_TOTALS2, RQ_TBASE, RQ_CAND, RQ_MARK, RQ_JUMP, RQ_ERRA, RQ_DPOS, RQ_DLEN, RQ_VER, RQ_OWN,
           RQ_SLOT, RQ_TABLE, RQ_NREC, RQ_NVER, RQ_NOWN, RQ_NPLEN, RQ_NDLEN, RQ_GTOT, RQ_PB, RQ_PO, RQ_JB, RQ_JO, RQ_COUNT,
           RQ_NBUF };
    DevBuf rq[RQ_NBUF];
    HostBuf h_rq_count, h_rq_err, h_rq_node;
    cudaEvent_t rq_ev[2] = {nullptr, nullptr};
    std::vector<cudaEvent_t> pipe_events;
    /* skip mode (regk_skip.cuh): fence workspace, the compacted batch, the expanded offsets, the skipped list */
    DevBuf skip_work, skip_in[11], skip_off_p, skip_off_j, skip_index, skip_bits;
    HostBuf h_skip_status, h_skip_index, h_skip_bits;
    struct SkipLast {
        bool valid = false;                     /* the batch finished last was a skip-mode batch */
        uint64_t n = 0, n_skipped = 0;
        uint32_t bad_bits = 0;
    } skip_last;
    /* workspace: DevStatus | two-level byte totals of both halves (stream-ordered reuse; host pipelining) */
    DevBuf work;
    /* device-resident batches rotate through a ring of workspaces that a side stream re-zeroes (and copies
       the status out of) after each use, so the main stream carries nothing but the two kernels */
    static constexpr int NWORK = 4;
    DevBuf work_ring[NWORK];
    cudaEvent_t ws_clean[NWORK] = {nullptr, nullptr, nullptr, nullptr};
    size_t ws_clean_bytes[NWORK] = {0, 0, 0, 0};
    cudaStream_t s_side = nullptr;
    uint64_t ws_seq = 0;

    /* in-flight batches: events + pinned status per slot.  Outputs are single-buffered: with the
       "async" option several batches may be enqueued back to back (benchmark loops), each one
       overwriting the previous batch's outputs in stream order. */
    struct Slot {
        cudaEvent_t ev[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};     /* [5]: after a job step's closing exchange */
        PathParams path_params{};               /* kept for the exact-offset redo (empty labels) */
        size_t path_smem = 0;
        bool path_alias = false, did_path = false;
        DevStatus *d_status = nullptr;
        DevStatus *h_status = nullptr;          /* pinned */
        int ring = -1;                          /* workspace ring entry used by this batch */
        int hset = -1;                          /* async host batch: which HostSet it lives in */
        bool d2h_issued = false;
        bool timed = true;                      /* ev[0..2] were recorded for this batch */
        const uint8_t *dev_path_bytes = nullptr;        /* where this batch's path stream lives on the device */
        const unsigned long long *dev_path_off = nullptr;
        const uint8_t *dev_json_bytes = nullptr;
        const unsigned long long *dev_json_off = nullptr;
        const uint32_t *dev_host_off = nullptr;         /* how its paths end: hostname lengths (NULL: fixed stride) */
        uint32_t host_stride = 0;
        bool alias = false;
        bool job = false;                       /* a REGK_JOB_STEP batch */
        bool off32 = false;                     /* host results with 32-bit offsets (option "offsets32") */
        uint64_t json_est = 0;                  /* a-priori payload bytes per record of this batch */
        bool json_learned = false;              /* its image budget came from json_mean_seen */
        bool in_use = false;
        uint64_t n = 0;
        uint32_t flags = 0;
        uint32_t launches = 0;
        /* REGK_SKIP_BAD: the batch's device inputs as its kernels read them, for the redo of a dirty batch */
        const void *dev_in[11] = {};
        uint64_t in_len[4] = {};                /* domain bytes, host bytes, address bytes, port elements */
        uint32_t in_stride = 0;
    };
    static constexpr int NSLOTS = 64;
    Slot slots[NSLOTS];
    DevStatus *h_status_block = nullptr;        /* pinned, NSLOTS entries */
    uint64_t seq = 0;
    int pending = 0;

    std::map<std::string, int64_t> opt;
};

namespace {

int fail(regk_ctx *c, int code, const char *fmt, ...)
{
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    if (c)
        c->err = buf;
    else
        g_create_error = buf;
    return code;
}

#define CK(call)                                                                                   \
    do {                                                                                           \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess)                                                                     \
            return fail(ctx, REGK_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), \
                __FILE__, __LINE__);                                                               \
    } while (0)

int ensure_dev(regk_ctx *ctx, DevBuf &b, size_t bytes)
{
    bytes = (bytes + 255) & ~(size_t)255;
    if (bytes <= b.cap)
        return REGK_OK;
    if (b.p)
        CK(cudaFree(b.p));
    b.p = nullptr;
    b.cap = 0;
    size_t want = bytes + bytes / 8;            /* a little slack so slowly growing batches do not thrash */
    cudaError_t e = cudaMalloc(&b.p, want);
    if (e != cudaSuccess) {
        cudaGetLastError();
        e = cudaMalloc(&b.p, bytes);
        want = bytes;
    }
    if (e != cudaSuccess)
        return fail(ctx, REGK_ERR_NOMEM, "cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
    b.cap = want;
    return REGK_OK;
}

int ensure_host(regk_ctx *ctx, HostBuf &b, size_t bytes)
{
    bytes = (bytes + 4095) & ~(size_t)4095;
    if (bytes <= b.cap)
        return REGK_OK;
    if (b.p)
        CK(cudaFreeHost(b.p));
    b.p = nullptr;
    b.cap = 0;
    cudaError_t e = cudaMallocHost(&b.p, bytes);
    if (e != cudaSuccess)
        return fail(ctx, REGK_ERR_NOMEM, "cudaMallocHost(%zu) failed: %s", bytes, cudaGetErrorString(e));
    b.cap = bytes;
    return REGK_OK;
}

int64_t opt_get(const regk_ctx *c, const char *name, int64_t dflt)
{
    auto it = c->opt.find(name);
    return it == c->opt.end() ? dflt : it->second;
}

size_t align16(size_t v)
{
    return (v + 15) & ~(size_t)15;
}

/* cudaFuncAttributeMaxDynamicSharedMemorySize is per function and device, shared by every context of the
   process: raise it monotonically and remember the high-water mark (which: 0 alias paths, 1 node paths, 2 payloads) */
bool smem_attr_needs_raise(int device, int which, size_t bytes)
{
    static std::mutex mu;
    static size_t high[64][4];
    std::lock_guard<std::mutex> lock(mu);
    size_t &h = high[device & 63][which];
    if (bytes <= h)
        return false;
    h = bytes;
    return true;
}

/* Lookahead distance of a compose kernel (PathParams / JsonParams::lookahead): half a wave, where a wave is how many
   of its CTAs the GPU holds at once with `smem` bytes of dynamic shared memory.  The tile that far ahead starts about
   half a CTA lifetime later, when its prefetched metadata has landed in L2.  On an H100, half a wave measured faster
   than one (DESIGN.md §4). */
int lookahead_tiles(regk_ctx *ctx, int which, const void *kernel, size_t smem, uint32_t *out)
{
    auto it = ctx->wave_ctas[which].find(smem);        /* batches of one workload alternate between a few budgets */
    if (it == ctx->wave_ctas[which].end()) {
        int per_sm = 0;
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, TILE, smem));
        it = ctx->wave_ctas[which].emplace(smem, (uint32_t)per_sm * (uint32_t)ctx->sm_count).first;
    }
    *out = it->second / 2;
    return REGK_OK;
}

}  // namespace

/* "offsets32": host results carry 32-bit offsets (half the D2H bytes of the two offset arrays) */
__global__ void __launch_bounds__(256) regk_off32_kernel(const unsigned long long *__restrict__ src, uint32_t *__restrict__ dst, uint64_t n1)
{
    const uint64_t i = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (i < n1)
        dst[i] = (uint32_t)src[i];
}

static int narrow_offsets(regk_ctx *ctx, const void *src64, DevBuf &dst32, uint64_t n, cudaStream_t s)
{
    int rc = ensure_dev(ctx, dst32, (n + 1) * 4);
    if (rc)
        return rc;
    regk_off32_kernel<<<(unsigned)((n + 1 + 255) / 256), 256, 0, s>>>((const unsigned long long *)src64, (uint32_t *)dst32.p, n + 1);
    CK(cudaGetLastError());
    return REGK_OK;
}

/*
 * Host buffers in, host buffers out, large batch: the PCIe copies dominate (config 2: 91 MB in, 171 MB out
 * per million records against ~0.12 ms of kernels), so the batch is cut into chunks of `chunk` records and
 * three streams overlap  H2D(chunk c+1) | kernels(chunk c) | D2H(chunk c-1).  Inputs land at their final
 * positions in whole-batch device arrays, so offsets stay absolute; a chunk's kernels get pointer-shifted
 * views, `off_bias` / `rec0` for the record numbering and a running payload base (device array) chained
 * from chunk to chunk.  The host learns each chunk's payload byte range from a pinned copy of that running
 * total once the chunk's kernels are done, then issues its D2H.
 */
struct HostPipe {
    uint64_t chunk = 0, nchunks = 0, nsuper_chunk = 0;
    unsigned long long *running = nullptr;      /* device, [nchunks + 1], zeroed */
    uint64_t path_cap = 0, json_cap = 0;
    const void *src[11] = {};
    void *dev[11] = {};
};

/* run_pipelined uses the caller's offsets at chunk boundaries as cudaMemcpyAsync byte ranges: every boundary
   must be monotone and inside the declared array (off[n]).  A batch that fails this takes the unpipelined path,
   whose kernels report the first offending record as REGK_BAD_TOO_LARGE without dereferencing anything. */
static bool chunk_bounds_ok(const regk_batch *b, uint64_t chunk, bool do_path, bool do_json, bool alias)
{
    const uint64_t n = b->n;
    auto ok = [&](const uint32_t *off) {
        if (!off)
            return true;
        uint32_t prev = off[0];
        const uint32_t last = off[n];
        if (prev != 0 && prev > last)
            return false;
        for (uint64_t r = chunk; r < n; r += chunk) {
            if (off[r] < prev || off[r] > last)
                return false;
            prev = off[r];
        }
        return true;
    };
    return (!do_path || (ok(b->domain_off) && (alias || ok(b->host_off)))) &&
           (!do_json || (ok(b->addr_off) && ok(b->ports_off)));
}

static int run_pipelined(regk_ctx *ctx, const regk_batch *b, regk_result *res, const PathParams &pp0, size_t path_smem,
    const JsonParams &jp0, size_t json_smem, const HostPipe &hp)
{
    const uint64_t n = b->n;
    const bool alias = b->flags & REGK_NODE_ALIAS;
    const bool do_path = !(b->flags & REGK_NO_PATH), do_json = !(b->flags & REGK_NO_JSON);
    const uint32_t stride = b->host_stride;
    cudaStream_t s = ctx->stream;
    int rc;
    if (!ctx->s_h2d) {
        CK(cudaStreamCreateWithFlags(&ctx->s_h2d, cudaStreamNonBlocking));
        CK(cudaStreamCreateWithFlags(&ctx->s_d2h, cudaStreamNonBlocking));
    }
    while (ctx->pipe_events.size() < 3 * hp.nchunks + 2) {
        cudaEvent_t e;
        CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        ctx->pipe_events.push_back(e);
    }
    if ((rc = ensure_host(ctx, ctx->h_path_bytes, hp.path_cap)) || (rc = ensure_host(ctx, ctx->h_path_off, (n + 1) * 8)) ||
        (rc = ensure_host(ctx, ctx->h_json_bytes, hp.json_cap)) || (rc = ensure_host(ctx, ctx->h_json_off, (n + 1) * 8)) ||
        (rc = ensure_host(ctx, ctx->h_running, (hp.nchunks + 2) * 8)))
        return rc;
    unsigned long long *h_running = (unsigned long long *)ctx->h_running.p;
    DevStatus *d_status = pp0.status ? pp0.status : jp0.status;
    DevStatus *h_status = ctx->slots[0].h_status;

    /* the workspace memset and the type table are ordered before everything on s */
    cudaEvent_t e_ready = ctx->pipe_events[3 * hp.nchunks];
    CK(cudaEventRecord(e_ready, s));
    CK(cudaStreamWaitEvent(ctx->s_h2d, e_ready, 0));

    const uint32_t *dom_off = (const uint32_t *)b->domain_off, *host_off = (const uint32_t *)b->host_off,
                   *addr_off = (const uint32_t *)b->addr_off, *ports_off = (const uint32_t *)b->ports_off;
    auto h2d = [&](int i, size_t byte_lo, size_t byte_hi) -> cudaError_t {
        if (!hp.src[i] || !hp.dev[i] || byte_hi <= byte_lo)
            return cudaSuccess;
        return cudaMemcpyAsync((uint8_t *)hp.dev[i] + byte_lo, (const uint8_t *)hp.src[i] + byte_lo, byte_hi - byte_lo,
            cudaMemcpyHostToDevice, ctx->s_h2d);
    };
    /* closed-form path offset of record r (no empty labels; verified by the kernel) */
    auto path_cf = [&](uint64_t r) -> uint64_t {
        if (alias)
            return (uint64_t)dom_off[r] + r;
        return (uint64_t)dom_off[r] + 2 * r + (host_off ? (uint64_t)host_off[r] : r * (uint64_t)stride);
    };

    uint32_t launches = 0;
    for (uint64_t c = 0; c < hp.nchunks; c++) {
        const uint64_t r0 = c * hp.chunk, r1 = std::min(n, r0 + hp.chunk), cn = r1 - r0;
        const uint64_t t0 = r0 / TILE, ct = (cn + TILE - 1) / TILE;
        cudaEvent_t e_in = ctx->pipe_events[3 * c], e_done = ctx->pipe_events[3 * c + 1];
        /* ---- H2D of this chunk's slices ---- */
        if (do_path) {
            CK(h2d(1, r0 * 4, (r1 + 1) * 4));
            CK(h2d(0, dom_off[r0], dom_off[r1]));
            if (!alias) {
                if (host_off) {
                    CK(h2d(3, r0 * 4, (r1 + 1) * 4));
                    CK(h2d(2, host_off[r0], host_off[r1]));
                } else {
                    CK(h2d(2, r0 * (size_t)stride, r1 * (size_t)stride));
                }
            }
        }
        if (do_json) {
            CK(h2d(4, r0, r1));
            CK(h2d(6, r0 * 4, (r1 + 1) * 4));
            CK(h2d(5, addr_off[r0], addr_off[r1]));
            CK(h2d(7, r0 * 4, r1 * 4));
            if (ports_off) {
                CK(h2d(8, r0 * 4, (r1 + 1) * 4));
                CK(h2d(9, (size_t)ports_off[r0] * 4, (size_t)ports_off[r1] * 4));
            }
            CK(h2d(10, r0, r1));
        }
        CK(cudaEventRecord(e_in, ctx->s_h2d));
        CK(cudaStreamWaitEvent(s, e_in, 0));
        /* ---- kernels on pointer-shifted views ---- */
        PathParams pp = pp0;
        JsonParams jp = jp0;
        if (do_json) {
            jp.n = cn;
            jp.rec0 = r0;
            jp.type_id += r0;
            jp.addr_off += r0;
            if (jp.ttl)
                jp.ttl += r0;
            if (jp.ports_off)
                jp.ports_off += r0;
            if (jp.ports_present)
                jp.ports_present += r0;
            jp.out_off += r0;
            jp.tile_total += t0;
            jp.super_total += c * hp.nsuper_chunk;
            jp.base_in = hp.running + c;
            jp.base_out = hp.running + c + 1;
        }
        if (do_path) {
            pp.n = cn;
            pp.rec0 = r0;
            pp.domain_off += r0;
            if (pp.host_off) {
                pp.host_off += r0;
                pp.off_bias = alias ? r0 : 2 * r0;
            } else if (!alias) {
                pp.host_bytes += r0 * (size_t)stride;
                pp.host_limit -= r0 * (uint64_t)stride;
                pp.off_bias = r0 * (uint64_t)(stride + 2);
            } else {
                pp.off_bias = r0;
            }
            pp.out_off += r0;
            pp.tile_total += t0;
            pp.super_total += c * hp.nsuper_chunk;
            const JsonParams side = do_json ? jp : JsonParams{};
            if (alias)
                regk_path_kernel<true, false><<<(unsigned)ct, TILE, path_smem, s>>>(pp, side);
            else
                regk_path_kernel<false, false><<<(unsigned)ct, TILE, path_smem, s>>>(pp, side);
            CK(cudaGetLastError());
            launches++;
        }
        if (do_json) {
            if (!do_path) {
                regk_json_len_kernel<<<(unsigned)std::min<uint64_t>(ct, (uint64_t)ctx->sm_count * 8), TILE, 0, s>>>(jp, (uint32_t)ct);
                CK(cudaGetLastError());
                launches++;
            }
            regk_json_kernel<<<(unsigned)ct, TILE, json_smem, s>>>(jp);
            CK(cudaGetLastError());
            launches++;
            CK(cudaMemcpyAsync(h_running + c + 1, hp.running + c + 1, 8, cudaMemcpyDeviceToHost, s));
        }
        if (c + 1 == hp.nchunks)
            CK(cudaMemcpyAsync(h_status, d_status, sizeof(DevStatus), cudaMemcpyDeviceToHost, s));
        CK(cudaEventRecord(e_done, s));
    }
    /* ---- D2H, chunk by chunk, as soon as each chunk's kernels are done ---- */
    h_running[0] = 0;
    for (uint64_t c = 0; c < hp.nchunks; c++) {
        const uint64_t r0 = c * hp.chunk, r1 = std::min(n, r0 + hp.chunk);
        cudaError_t e = cudaEventSynchronize(ctx->pipe_events[3 * c + 1]);
        if (e != cudaSuccess)
            return fail(ctx, REGK_ERR_CUDA, "kernel execution failed: %s", cudaGetErrorString(e));
        const bool last = c + 1 == hp.nchunks;
        if (do_path) {
            const uint64_t lo = path_cf(r0), hi = std::min<uint64_t>(path_cf(r1), hp.path_cap);
            if (hi > lo)
                CK(cudaMemcpyAsync((uint8_t *)ctx->h_path_bytes.p + lo, (uint8_t *)ctx->path_bytes.p + lo, hi - lo,
                    cudaMemcpyDeviceToHost, ctx->s_d2h));
            CK(cudaMemcpyAsync((uint64_t *)ctx->h_path_off.p + r0, (uint64_t *)ctx->path_off.p + r0, (r1 - r0 + (last ? 1 : 0)) * 8,
                cudaMemcpyDeviceToHost, ctx->s_d2h));
        }
        if (do_json) {
            const uint64_t lo = h_running[c], hi = std::min<uint64_t>(h_running[c + 1], hp.json_cap);
            if (hi > lo)
                CK(cudaMemcpyAsync((uint8_t *)ctx->h_json_bytes.p + lo, (uint8_t *)ctx->json_bytes.p + lo, hi - lo,
                    cudaMemcpyDeviceToHost, ctx->s_d2h));
            CK(cudaMemcpyAsync((uint64_t *)ctx->h_json_off.p + r0, (uint64_t *)ctx->json_off.p + r0, (r1 - r0 + (last ? 1 : 0)) * 8,
                cudaMemcpyDeviceToHost, ctx->s_d2h));
        }
    }
    cudaError_t e = cudaStreamSynchronize(ctx->s_d2h);
    if (e != cudaSuccess)
        return fail(ctx, REGK_ERR_CUDA, "device-to-host copy failed: %s", cudaGetErrorString(e));
    const DevStatus st = *h_status;
    memset(res, 0, sizeof *res);
    res->n = n;
    res->launches = launches;
    res->bad_bits = st.bad_bits;
    res->first_bad = st.bad_bits ? ~st.first_bad : 0;
    if (st.overflow)
        return fail(ctx, REGK_ERR_CUDA, "internal error: output capacity bound exceeded");
    if (st.bad_bits)
        return fail(ctx, REGK_ERR_OUT_OF_DOMAIN,
            "record %llu is outside the supported input domain (REGK_BAD bits 0x%x); no output produced",
            (unsigned long long)res->first_bad, st.bad_bits);
    if (st.needs_exact)
        return REGK_ERR_STATE + 100;            /* caller re-runs the batch through the exact-capable path */
    res->path_total = st.path_total;
    res->json_total = st.json_total;
    res->path_bytes = (uint8_t *)ctx->h_path_bytes.p;
    res->path_off = (uint64_t *)ctx->h_path_off.p;
    res->json_bytes = (uint8_t *)ctx->h_json_bytes.p;
    res->json_off = (uint64_t *)ctx->h_json_off.p;
    if (!do_path)
        memset(res->path_off, 0, (n + 1) * 8);
    if (!do_json)
        memset(res->json_off, 0, (n + 1) * 8);
    return REGK_OK;
}

/*
 * D2H of an async host batch into its set's pinned result buffers, on the D2H stream.  Called once the
 * batch's status has reached the host (its kernels are done), so the exact byte counts are known; a batch
 * that failed the fence or still needs the exact-offset redo is left to regk_finish.
 */
static int issue_d2h(regk_ctx *ctx, regk_ctx::Slot &slot)
{
    const DevStatus st = *slot.h_status;
    regk_ctx::HostSet &hs = ctx->hset[slot.hset];
    if (st.bad_bits || st.overflow)
        return REGK_OK;
    if (st.needs_exact && slot.did_path)
        return REGK_OK;
    const uint64_t n = slot.n;
    const bool do_path = !(slot.flags & REGK_NO_PATH), do_json = !(slot.flags & REGK_NO_JSON);
    int rc;
    if ((rc = ensure_host(ctx, hs.h_path_bytes, st.path_total + 16)) || (rc = ensure_host(ctx, hs.h_path_off, (n + 1) * 8)) ||
        (rc = ensure_host(ctx, hs.h_json_bytes, st.json_total + 16)) || (rc = ensure_host(ctx, hs.h_json_off, (n + 1) * 8)))
        return rc;
    cudaStream_t sd = ctx->s_d2h;
    slot.off32 = slot.off32 && st.path_total < (1ull << 32) && st.json_total < (1ull << 32);   /* else: 64-bit after all */
    const size_t ow = slot.off32 ? 4 : 8;
    if (n && do_path) {
        CK(cudaMemcpyAsync(hs.h_path_bytes.p, hs.path_bytes.p, st.path_total, cudaMemcpyDeviceToHost, sd));
        CK(cudaMemcpyAsync(hs.h_path_off.p, slot.off32 ? hs.off32_p.p : hs.path_off.p, (n + 1) * ow, cudaMemcpyDeviceToHost, sd));
    } else {
        memset(hs.h_path_off.p, 0, (n + 1) * 8);
    }
    if (n && do_json) {
        CK(cudaMemcpyAsync(hs.h_json_bytes.p, hs.json_bytes.p, st.json_total, cudaMemcpyDeviceToHost, sd));
        CK(cudaMemcpyAsync(hs.h_json_off.p, slot.off32 ? hs.off32_j.p : hs.json_off.p, (n + 1) * ow, cudaMemcpyDeviceToHost, sd));
    } else {
        memset(hs.h_json_off.p, 0, (n + 1) * 8);
    }
    CK(cudaEventRecord(hs.e_out, sd));
    slot.d2h_issued = true;
    return REGK_OK;
}

template <bool MULTI, bool DATA>
static cudaError_t launch_jute(const JuteParams &p, size_t smem, int device, cudaStream_t s)
{
    static std::mutex mu;
    static size_t high[64];
    {
        std::lock_guard<std::mutex> lock(mu);
        if (smem > high[device & 63]) {
            cudaError_t e = cudaFuncSetAttribute(regk_jute_kernel<MULTI, DATA>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e != cudaSuccess)
                return e;
            high[device & 63] = smem;
        }
    }
    regk_jute_kernel<MULTI, DATA><<<(unsigned)((p.n + JUTE_TILE - 1) / JUTE_TILE), JUTE_THREADS, smem, s>>>(p);
    return cudaGetLastError();
}

/* The request frames of one (path, payload) stream pair on the device - regk_jute_requests on the batch finished last,
   regk_mkdirp_requests on the mkdirp set - into the given buffers.  json_off == NULL: no data (delete). */
struct FrameSrc {
    uint64_t n;
    const uint8_t *path_bytes;
    const unsigned long long *path_off;
    const uint8_t *json_bytes;
    const unsigned long long *json_off;
    const char *who = "regk_jute_requests";
};

/* What the framing driver hands a framing kernel: the streams' extents, the output buffers, the staging budgets. */
struct FrameGeom {
    uint64_t n, total;
    uint8_t *out_bytes;
    unsigned long long *out_off;
    DevStatus *status;
    uint32_t path_cap, json_cap;
    uint64_t path_limit, json_limit;
    size_t smem;
};

/* The driver both framing kernels share: read the streams' totals, size and fill the buffers, launch (`launch` fills the
   kernel's own parameters from the geometry), check the status, copy the frames out.  Frames are multi transactions of
   `group` entries when `multi`, else one request per entry; every entry carries `per_rec` framing bytes, emits its path
   `path_times` times, and a tile's framing slots take `slot_bytes` of shared memory. */
static int frame_drive(regk_ctx *ctx, const FrameSrc &src, const regk_jute_opts *o, bool multi, uint64_t group, uint32_t per_rec,
    uint32_t path_times, size_t slot_bytes, DevBuf &db, DevBuf &doff, HostBuf &hb, HostBuf &hoff, regk_frames *out,
    const std::function<cudaError_t(const FrameGeom &)> &launch)
{
    const uint64_t n = src.n;
    const bool has_data = src.json_off != nullptr;
    const uint64_t frames = (n + group - 1) / group;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    const bool dev_out = o->flags & REGK_OUT_DEVICE;
    out->n = frames;
    out->flags = dev_out ? REGK_OUT_DEVICE : 0;
    /* totals of the two streams: the closing offsets on the device */
    unsigned long long tot[2] = {0, 0};
    CK(cudaMemcpyAsync(&tot[0], src.path_off + n, 8, cudaMemcpyDeviceToHost, s));
    if (has_data)
        CK(cudaMemcpyAsync(&tot[1], src.json_off + n, 8, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    const uint64_t total = path_times * tot[0] + tot[1] + (uint64_t)per_rec * n + (uint64_t)JUTE_FRAME_HEAD * frames +
        (multi ? (uint64_t)JUTE_MULTI_HEAD * frames : 0);
    int rc;
    if ((rc = ensure_dev(ctx, db, total + 32)) || (rc = ensure_dev(ctx, doff, (frames + 1) * 8)))
        return rc;
    if ((rc = ensure_dev(ctx, ctx->svc_work, 256)))
        return rc;
    CK(cudaMemsetAsync(ctx->svc_work.p, 0, sizeof(DevStatus), s));
    if (n == 0)
        CK(cudaMemsetAsync(doff.p, 0, 8, s));
    cudaEvent_t e0 = ctx->slots[0].ev[0], e1 = ctx->slots[0].ev[1];
    if (n) {
        FrameGeom g{};
        g.n = n;
        g.total = total;
        g.out_bytes = (uint8_t *)db.p;
        g.out_off = (unsigned long long *)doff.p;
        g.status = (DevStatus *)ctx->svc_work.p;
        /* staging budgets: 9/8 of a tile's mean share of each stream plus slack (tiles beyond it go byte-wise) */
        g.path_cap = (uint32_t)align16(std::min<uint64_t>(tot[0] * JUTE_TILE / n * 9 / 8 + 1024, 65520));
        g.json_cap = has_data ? (uint32_t)align16(std::min<uint64_t>(tot[1] * JUTE_TILE / n * 9 / 8 + 1024, 65520)) : 0u;  /* lengths travel as 16 bits */
        g.path_limit = tot[0] + 16;                 /* every stream buffer of this library has >= 16 bytes of slack */
        g.json_limit = has_data ? tot[1] + 16 : 0;
        /* ... + one owner byte and one list entry per 16-byte output block of a tile that fits the staging budgets */
        const uint32_t max_fixed = per_rec + JUTE_FRAME_HEAD + JUTE_MULTI_HEAD;
        const size_t owner_bytes = 3 * ((path_times * g.path_cap + g.json_cap + max_fixed * JUTE_TILE) / 16 + 32);   /* owner u8 + list u16 per block */
        g.smem = 34 * 16 + 16 + slot_bytes + 16 + (size_t)g.path_cap + 16 + g.json_cap + 48 + owner_bytes;
        CK(cudaEventRecord(e0, s));
        CK(launch(g));
        CK(cudaEventRecord(e1, s));
        out->launches = 1;
    }
    CK(cudaMemcpyAsync(ctx->slots[0].h_status, ctx->svc_work.p, sizeof(DevStatus), cudaMemcpyDeviceToHost, s));
    cudaError_t e = cudaStreamSynchronize(s);
    if (e != cudaSuccess)
        return fail(ctx, REGK_ERR_CUDA, "%s: kernel execution failed: %s", src.who, cudaGetErrorString(e));
    if (ctx->slots[0].h_status->overflow)
        return fail(ctx, REGK_ERR_CUDA, "internal error: frame capacity bound exceeded");
    if (n)
        cudaEventElapsedTime(&out->kernel_ms, e0, e1);
    out->total = total;
    if (dev_out) {
        out->frame_bytes = (const uint8_t *)db.p;
        out->frame_off = (const uint64_t *)doff.p;
        return REGK_OK;
    }
    if ((rc = ensure_host(ctx, hb, total + 16)) || (rc = ensure_host(ctx, hoff, (frames + 1) * 8)))
        return rc;
    if (total)
        CK(cudaMemcpyAsync(hb.p, db.p, total, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(hoff.p, doff.p, (frames + 1) * 8, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    out->frame_bytes = (const uint8_t *)hb.p;
    out->frame_off = (const uint64_t *)hoff.p;
    return REGK_OK;
}

static int frame_requests(regk_ctx *ctx, const FrameSrc &src, const regk_jute_opts *o, DevBuf &db, DevBuf &doff, HostBuf &hb,
    HostBuf &hoff, regk_frames *out)
{
    const bool has_data = src.json_off != nullptr;
    const bool multi = o->group != 0;
    const uint64_t g = multi ? o->group : 1;
    JuteParams p{};
    p.n = src.n;
    p.op = o->op;
    p.mid = has_data ? 4u : 0u;
    p.group = (uint32_t)g;
    p.multi = multi ? 1u : 0u;
    /* what follows the data: create - acl vector [OPEN_ACL_UNSAFE] + flags; delete / setData - the expected version */
    uint8_t tail[48] = {0};
    if (o->op == REGK_ZK_GETDATA) {
        p.tail_len = 1;                                 /* watch = false */
    } else if (o->op == REGK_ZK_CREATE) {
        static const uint8_t acl[27] = {0, 0, 0, 1, 0, 0, 0, 31, 0, 0, 0, 5, 'w', 'o', 'r', 'l', 'd', 0, 0, 0, 6, 'a', 'n', 'y', 'o', 'n', 'e'};
        memcpy(tail, acl, 27);
        for (int k = 0; k < 4; k++)
            tail[27 + k] = (uint8_t)(o->zk_flags >> (24 - 8 * k));
        p.tail_len = 31;
    } else {
        for (int k = 0; k < 4; k++)
            tail[k] = (uint8_t)((uint32_t)o->version >> (24 - 8 * k));
        p.tail_len = 4;
    }
    static const uint8_t multi_end[9] = {0xFF, 0xFF, 0xFF, 0xFF, 1, 0xFF, 0xFF, 0xFF, 0xFF};   /* MultiHeader {type -1, done, err -1} */
    memcpy(tail + p.tail_len, multi_end, 9);
    memcpy(p.tail, tail, sizeof p.tail);
    p.per_rec = (multi ? JUTE_MULTI_HEAD : 0u) + 4u + p.mid + p.tail_len;
    p.path_bytes = src.path_bytes;
    p.path_off = src.path_off;
    p.json_bytes = src.json_bytes;
    p.json_off = src.json_off;
    p.xid_base = o->xid_base;
    /* framing slots, 16 bytes of slack, the constant tail */
    const size_t slot_bytes = JUTE_TILE * JUTE_SLOT + 16 + 48;
    return frame_drive(ctx, src, o, multi, g, p.per_rec, 1, slot_bytes, db, doff, hb, hoff, out, [&](const FrameGeom &G) {
        p.out_bytes = G.out_bytes;
        p.out_off = G.out_off;
        p.out_capacity = G.total;
        p.status = G.status;
        p.path_cap = G.path_cap;
        p.json_cap = G.json_cap;
        p.path_limit = G.path_limit;
        p.json_limit = G.json_limit;
        return multi ? (has_data ? launch_jute<true, true>(p, G.smem, ctx->device, ctx->stream)
                                 : launch_jute<true, false>(p, G.smem, ctx->device, ctx->stream))
                     : (has_data ? launch_jute<false, true>(p, G.smem, ctx->device, ctx->stream)
                                 : launch_jute<false, false>(p, G.smem, ctx->device, ctx->stream));
    });
}

template <bool MULTI, bool DATA, bool PAIR>
static cudaError_t launch_jute_entry(const JuteEntryParams &p, size_t smem, int device, cudaStream_t s)
{
    static std::mutex mu;
    static size_t high[64];
    {
        std::lock_guard<std::mutex> lock(mu);
        if (smem > high[device & 63]) {
            cudaError_t e = cudaFuncSetAttribute(regk_jute_entry_kernel<MULTI, DATA, PAIR>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                 (int)smem);
            if (e != cudaSuccess)
                return e;
            high[device & 63] = smem;
        }
    }
    regk_jute_entry_kernel<MULTI, DATA, PAIR><<<(unsigned)((p.n + JUTE_TILE - 1) / JUTE_TILE), JUTE_THREADS, smem, s>>>(p);
    return cudaGetLastError();
}

/* Frames whose entries carry a version of their own (`version`: [n] device array, NULL = o->version for all) or that
   pair a delete with a create (`pair`: REGK_ZK_REPLACE, always multi transactions) - regk_jute_entry_kernel.  Output
   and buffers as frame_requests. */
static int frame_entry_requests(regk_ctx *ctx, const FrameSrc &src, const regk_jute_opts *o, const int32_t *version, bool pair,
    DevBuf &db, DevBuf &doff, HostBuf &hb, HostBuf &hoff, regk_frames *out)
{
    const bool has_data = src.json_off != nullptr;
    const bool multi = pair || o->group != 0;
    const uint64_t g = o->group ? o->group : 1;
    JuteEntryParams p{};
    p.n = src.n;
    p.op = pair ? (uint32_t)REGK_ZK_DELETE : o->op;
    p.zk_flags = o->zk_flags;
    p.version = version;
    p.version_const = o->version;
    p.group = (uint32_t)g;
    /* delete: path length + version; setData: + data length; replace: 17 + P + 4 + J + 31 around the paths and data */
    p.per_rec = (multi ? JUTE_MULTI_HEAD : 0u) + 4u + (pair ? 17u : 0u) + (has_data ? 4u : 0u) + (pair ? 31u : 4u);
    p.path_bytes = src.path_bytes;
    p.path_off = src.path_off;
    p.json_bytes = src.json_bytes;
    p.json_off = src.json_off;
    p.xid_base = o->xid_base;
    return frame_drive(ctx, src, o, multi, g, p.per_rec, pair ? 2 : 1, JUTE_TILE * JUTE_ESLOT, db, doff, hb, hoff, out,
        [&](const FrameGeom &G) {
            p.out_bytes = G.out_bytes;
            p.out_off = G.out_off;
            p.out_capacity = G.total;
            p.status = G.status;
            p.path_cap = G.path_cap;
            p.json_cap = G.json_cap;
            p.path_limit = G.path_limit;
            p.json_limit = G.json_limit;
            cudaStream_t s = ctx->stream;
            return pair ? launch_jute_entry<true, true, true>(p, G.smem, ctx->device, s)
                : multi ? (has_data ? launch_jute_entry<true, true, false>(p, G.smem, ctx->device, s)
                                    : launch_jute_entry<true, false, false>(p, G.smem, ctx->device, s))
                        : (has_data ? launch_jute_entry<false, true, false>(p, G.smem, ctx->device, s)
                                    : launch_jute_entry<false, false, false>(p, G.smem, ctx->device, s));
        });
}

/* regk_parents.cuh on the path stream of the batch finished last (n >= 1 records), into the given buffers: enqueues
   the table reset, `start` (if any) and the three kernels on the context's stream; p->parent_len / unique_first / n_unique are device
   pointers into `len` and `unique`. */
static int enqueue_parent_pass(regk_ctx *ctx, DevBuf &len, DevBuf &slot, DevBuf &table, DevBuf &totals, DevBuf &unique, uint64_t n,
    cudaEvent_t start, ParentParams *out)
{
    cudaStream_t s = ctx->stream;
    uint64_t slots = 1024;
    while (slots < 2 * n)
        slots <<= 1;
    const uint64_t ntiles = (n + PARENT_TILE - 1) / PARENT_TILE;
    const size_t totals_bytes = ((ntiles * 4 + 15) & ~(size_t)15) + (ntiles / SUPER + 1) * 8 + 16;
    int rc;
    if ((rc = ensure_dev(ctx, len, n * 4)) || (rc = ensure_dev(ctx, slot, n * 4)) || (rc = ensure_dev(ctx, table, slots * 4)) ||
        (rc = ensure_dev(ctx, totals, totals_bytes)) || (rc = ensure_dev(ctx, unique, n * 8 + 8)))
        return rc;
    ParentParams p{};
    p.n = n;
    p.path_bytes = ctx->last_path_bytes;
    p.path_off = ctx->last_path_off;
    p.parent_len = (uint32_t *)len.p;
    p.slot_of = (uint32_t *)slot.p;
    p.owner = (uint32_t *)table.p;
    p.mask = (uint32_t)(slots - 1);
    p.tile_total = (uint32_t *)totals.p;
    p.super_total = (unsigned long long *)((uint8_t *)totals.p + ((ntiles * 4 + 15) & ~(size_t)15));
    p.unique_first = (unsigned long long *)unique.p;
    p.n_unique = p.unique_first + n;
    p.tail_mode = ctx->last_alias ? 0u : (ctx->last_host_off ? 2u : 1u);
    p.host_stride = ctx->last_host_stride;
    p.host_off = ctx->last_host_off;
    CK(cudaMemsetAsync(p.owner, 0, slots * 4, s));
    CK(cudaMemsetAsync(totals.p, 0, totals_bytes, s));
    if (start)
        CK(cudaEventRecord(start, s));                  /* the kernels' time starts here */
    regk_parent_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(p);
    regk_parent_mark_kernel<<<(unsigned)ntiles, PARENT_TILE, 0, s>>>(p);
    regk_parent_compact_kernel<<<(unsigned)ntiles, PARENT_TILE, 0, s>>>(p);
    CK(cudaGetLastError());
    *out = p;
    return REGK_OK;
}

extern "C" {

int regk_abi_version(void)
{
    return REGK_ABI_VERSION;
}

const char *regk_last_error(const regk_ctx *ctx)
{
    return ctx ? ctx->err.c_str() : g_create_error.c_str();
}

int regk_create(int device, regk_ctx **out)
{
    regk_ctx *ctx = nullptr;
    if (!out)
        return fail(nullptr, REGK_ERR_INVALID_ARG, "regk_create: out is NULL");
    *out = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return fail(nullptr, REGK_ERR_CUDA, "regk_create: no CUDA device (%s); this library has no CPU fallback",
            e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0");
    if (device < 0 || device >= ndev)
        return fail(nullptr, REGK_ERR_INVALID_ARG, "regk_create: device %d out of range (0..%d)", device, ndev - 1);
    ctx = new regk_ctx();
    ctx->device = device;
#define CKC(call)                                                                               \
    do {                                                                                        \
        cudaError_t e_ = (call);                                                                \
        if (e_ != cudaSuccess) {                                                                \
            int rc_ = fail(nullptr, REGK_ERR_CUDA, "%s failed: %s", #call, cudaGetErrorString(e_)); \
            delete ctx;                                                                         \
            return rc_;                                                                         \
        }                                                                                       \
    } while (0)
    CKC(cudaSetDevice(device));
    cudaDeviceProp prop;
    CKC(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {   /* sm_90a code runs on compute capability 9.0 only */
        int rc = fail(nullptr, REGK_ERR_CUDA, "regk_create: device %d is sm_%d%d; this build targets sm_90a (H100)",
            device, prop.major, prop.minor);
        delete ctx;
        return rc;
    }
    ctx->sm_count = prop.multiProcessorCount;
    ctx->max_smem_optin = (int)prop.sharedMemPerBlockOptin;
    CKC(cudaStreamCreateWithFlags(&ctx->own_stream, cudaStreamNonBlocking));
    ctx->stream = ctx->own_stream;
    CKC(cudaMallocHost((void **)&ctx->h_status_block, sizeof(DevStatus) * regk_ctx::NSLOTS));
    memset(ctx->h_status_block, 0, sizeof(DevStatus) * regk_ctx::NSLOTS);
    for (int i = 0; i < regk_ctx::NSLOTS; i++) {
        for (auto &ev : ctx->slots[i].ev)
            CKC(cudaEventCreate(&ev));
        ctx->slots[i].h_status = ctx->h_status_block + i;
    }
#undef CKC
    *out = ctx;
    return REGK_OK;
}

void regk_destroy(regk_ctx *ctx)
{
    if (!ctx)
        return;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    for (auto &b : ctx->in)
        if (b.p)
            cudaFree(b.p);
    for (DevBuf *b : {&ctx->blob_dev, &ctx->path_bytes, &ctx->path_off, &ctx->json_bytes, &ctx->json_off, &ctx->work, &ctx->off32_p,
             &ctx->off32_j})
        if (b->p)
            cudaFree(b->p);
    for (cudaEvent_t e : ctx->pipe_events)
        cudaEventDestroy(e);
    if (ctx->s_h2d)
        cudaStreamSynchronize(ctx->s_h2d);
    if (ctx->s_d2h)
        cudaStreamSynchronize(ctx->s_d2h);
    for (auto &hs : ctx->hset) {
        for (auto &b : hs.in)
            if (b.p)
                cudaFree(b.p);
        for (DevBuf *b : {&hs.path_bytes, &hs.path_off, &hs.json_bytes, &hs.json_off, &hs.off32_p, &hs.off32_j})
            if (b->p)
                cudaFree(b->p);
        for (HostBuf *b : {&hs.h_path_bytes, &hs.h_path_off, &hs.h_json_bytes, &hs.h_json_off})
            if (b->p)
                cudaFreeHost(b->p);
        if (hs.e_in)
            cudaEventDestroy(hs.e_in);
        if (hs.e_out)
            cudaEventDestroy(hs.e_out);
    }
    for (auto &e : ctx->ws_clean)
        if (e)
            cudaEventDestroy(e);
    for (auto &wb : ctx->work_ring)
        if (wb.p)
            cudaFree(wb.p);
    if (ctx->s_side)
        cudaStreamDestroy(ctx->s_side);
    if (ctx->s_h2d)
        cudaStreamDestroy(ctx->s_h2d);
    if (ctx->s_d2h)
        cudaStreamDestroy(ctx->s_d2h);
    for (HostBuf *b : {&ctx->h_path_bytes, &ctx->h_path_off, &ctx->h_json_bytes, &ctx->h_json_off, &ctx->h_running})
        if (b->p)
            cudaFreeHost(b->p);
    if (ctx->h_status_block)
        cudaFreeHost(ctx->h_status_block);
    if (ctx->h_gather_flag)
        cudaFreeHost(ctx->h_gather_flag);
    if (ctx->h_job_bases)
        cudaFreeHost(ctx->h_job_bases);
    if (ctx->job_bases.p)
        cudaFree(ctx->job_bases.p);
    for (auto &b : ctx->dec_in)
        if (b.p)
            cudaFree(b.p);
    for (DevBuf *b : {&ctx->dec_rec, &ctx->dec_dom, &ctx->dec_ports})
        if (b->p)
            cudaFree(b->p);
    for (HostBuf *b : {&ctx->h_jute_bytes, &ctx->h_jute_off, &ctx->h_dec_rec, &ctx->h_dec_dom, &ctx->h_dec_ports})
        if (b->p)
            cudaFreeHost(b->p);
    for (DevBuf *b : {&ctx->par_len, &ctx->par_slot, &ctx->par_table, &ctx->par_totals, &ctx->par_unique, &ctx->svc_work,
             &ctx->jute_bytes, &ctx->jute_off})
        if (b->p)
            cudaFree(b->p);
    for (auto &b : ctx->svc_in)
        if (b.p)
            cudaFree(b.p);
    for (auto &ev : ctx->par_ev)
        if (ev)
            cudaEventDestroy(ev);
    for (HostBuf *b : {&ctx->h_par_len, &ctx->h_par_unique, &ctx->h_par_count, &ctx->h_skip_status, &ctx->h_skip_index,
             &ctx->h_skip_bits})
        if (b->p)
            cudaFreeHost(b->p);
    for (auto &b : ctx->skip_in)
        if (b.p)
            cudaFree(b.p);
    for (DevBuf *b : {&ctx->skip_work, &ctx->skip_off_p, &ctx->skip_off_j, &ctx->skip_index, &ctx->skip_bits})
        if (b->p)
            cudaFree(b->p);
    for (auto &b : ctx->mk)
        if (b.p)
            cudaFree(b.p);
    for (HostBuf *b : {&ctx->h_mk_count, &ctx->h_mk_drec, &ctx->h_mk_dlen, &ctx->h_mk_dbytes, &ctx->h_mk_doff, &ctx->h_mk_depth,
             &ctx->h_mk_invalid, &ctx->h_mk_fbytes, &ctx->h_mk_foff})
        if (b->p)
            cudaFreeHost(b->p);
    for (auto &ev : ctx->mk_ev)
        if (ev)
            cudaEventDestroy(ev);
    for (auto &b : ctx->rc)
        if (b.p)
            cudaFree(b.p);
    for (HostBuf *b : {&ctx->h_rc_count, &ctx->h_rc_cls, &ctx->h_rc_match, &ctx->h_rc_obscls, &ctx->h_rc_fbytes, &ctx->h_rc_foff})
        if (b->p)
            cudaFreeHost(b->p);
    for (auto &b : ctx->h_rc_list)
        if (b.p)
            cudaFreeHost(b.p);
    for (auto &ev : ctx->rc_ev)
        if (ev)
            cudaEventDestroy(ev);
    for (auto &b : ctx->rq)
        if (b.p)
            cudaFree(b.p);
    for (HostBuf *b : {&ctx->h_rq_count, &ctx->h_rq_err, &ctx->h_rq_node})
        if (b->p)
            cudaFreeHost(b->p);
    for (auto &ev : ctx->rq_ev)
        if (ev)
            cudaEventDestroy(ev);
    for (auto &sl : ctx->slots)
        for (auto &ev : sl.ev)
            if (ev)
                cudaEventDestroy(ev);
    if (ctx->own_stream)
        cudaStreamDestroy(ctx->own_stream);
    delete ctx;
}

int regk_set_stream(regk_ctx *ctx, void *cuda_stream)
{
    if (!ctx)
        return REGK_ERR_INVALID_ARG;
    if (ctx->pending)
        return fail(ctx, REGK_ERR_STATE, "regk_set_stream: a batch is still pending; call regk_finish first");
    ctx->stream = cuda_stream ? (cudaStream_t)cuda_stream : ctx->own_stream;
    return REGK_OK;
}

int regk_set_option(regk_ctx *ctx, const char *name, int64_t value)
{
    if (!ctx || !name)
        return REGK_ERR_INVALID_ARG;
    static const char *known[] = {"async", "force_generic", "dom_cap", "json_out_cap", "chunk_records", "time_every", "offsets32",
                                  "mkdirp_tight_table", "reconcile_tight_table", nullptr};
    for (const char **k = known; *k; k++)
        if (!strcmp(*k, name)) {
            ctx->opt[name] = value;
            return REGK_OK;
        }
    return fail(ctx, REGK_ERR_INVALID_ARG, "regk_set_option: unknown option '%s'", name);
}

int64_t regk_get_option(const regk_ctx *ctx, const char *name)
{
    if (!ctx || !name)
        return -1;
    if (!strcmp(name, "sm_count"))
        return ctx->sm_count;
    return opt_get(ctx, name, 0);
}

int regk_set_types(regk_ctx *ctx, const char *const *types, const uint32_t *lens, uint32_t ntypes)
{
    if (!ctx || (!types && ntypes))
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_set_types: NULL argument");
    if (ntypes > 255)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_set_types: at most 255 types (type_id is one byte)");
    if (ctx->pending)
        return fail(ctx, REGK_ERR_STATE, "regk_set_types: a batch is still pending");
    CK(cudaSetDevice(ctx->device));
    std::vector<std::string> raw(ntypes);
    for (uint32_t i = 0; i < ntypes; i++)
        raw[i].assign(types[i], lens ? lens[i] : strlen(types[i]));
    std::vector<uint8_t> blob;
    uint32_t maxq = 0;
    std::string why;
    const int brc = build_type_blob(raw, &blob, &maxq, &why);
    if (brc)
        return fail(ctx, brc == 1 ? REGK_ERR_OUT_OF_DOMAIN : REGK_ERR_INVALID_ARG, "regk_set_types: %s", why.c_str());
    int rc = ensure_dev(ctx, ctx->blob_dev, blob.size());
    if (rc)
        return rc;
    CK(cudaMemcpyAsync(ctx->blob_dev.p, blob.data(), blob.size(), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->types = raw;
    ctx->blob_host = blob;
    ctx->max_type_q = maxq;
    ctx->json_mean_seen = 0.0;
    ctx->json_learning = true;
    return REGK_OK;
}

void *regk_host_alloc(regk_ctx *ctx, size_t bytes)
{
    if (!ctx)
        return nullptr;
    void *p = nullptr;
    cudaSetDevice(ctx->device);
    if (cudaMallocHost(&p, bytes ? bytes : 1) != cudaSuccess) {
        cudaGetLastError();
        return nullptr;
    }
    return p;
}

void regk_host_free(regk_ctx *ctx, void *p)
{
    (void)ctx;
    if (p)
        cudaFreeHost(p);
}

void *regk_dev_alloc(regk_ctx *ctx, size_t bytes)
{
    if (!ctx)
        return nullptr;
    void *p = nullptr;
    cudaSetDevice(ctx->device);
    if (cudaMalloc(&p, bytes ? bytes : 1) != cudaSuccess) {
        cudaGetLastError();
        return nullptr;
    }
    return p;
}

void regk_dev_free(regk_ctx *ctx, void *p)
{
    (void)ctx;
    if (p)
        cudaFree(p);
}

int regk_memcpy_h2d(regk_ctx *ctx, void *dst_dev, const void *src_host, size_t bytes)
{
    if (!ctx)
        return REGK_ERR_INVALID_ARG;
    CK(cudaSetDevice(ctx->device));
    CK(cudaMemcpyAsync(dst_dev, src_host, bytes, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return REGK_OK;
}

int regk_memcpy_d2h(regk_ctx *ctx, void *dst_host, const void *src_dev, size_t bytes)
{
    if (!ctx)
        return REGK_ERR_INVALID_ARG;
    CK(cudaSetDevice(ctx->device));
    CK(cudaMemcpyAsync(dst_host, src_dev, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return REGK_OK;
}

#ifdef REGK_PHASE_STAMPS
/* development build only (tools/tile_phases.py): from now on thread 0 of every compose CTA of this context's device
   stores its phase stamps into `dev_buf`, u64[2][tiles][8] (kernel, tile, {start, 4 phases, -, -, SM}); NULL stops */
int regk_phase_stamps(regk_ctx *ctx, void *dev_buf, uint64_t tiles)
{
    if (!ctx)
        return REGK_ERR_INVALID_ARG;
    CK(cudaSetDevice(ctx->device));
    CK(cudaStreamSynchronize(ctx->stream));
    unsigned long long *p = (unsigned long long *)dev_buf;
    const unsigned long long cap = dev_buf ? tiles : 0;
    CK(cudaMemcpyToSymbol(regk::g_phase_buf, &p, sizeof(p)));
    CK(cudaMemcpyToSymbol(regk::g_phase_cap, &cap, sizeof(cap)));
    return REGK_OK;
}
#endif

int regk_sync(regk_ctx *ctx)
{
    if (!ctx)
        return REGK_ERR_INVALID_ARG;
    CK(cudaSetDevice(ctx->device));
    CK(cudaStreamSynchronize(ctx->stream));
    if (ctx->h_gather_flag && *ctx->h_gather_flag) {
        *ctx->h_gather_flag = 0;
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_gather_push: the totals table exceeds the whole-job buffers or disagrees with the shard; nothing was stored");
    }
    return REGK_OK;
}

int regk_ipc_export(regk_ctx *ctx, const void *dev_ptr, unsigned char handle[REGK_IPC_HANDLE_BYTES])
{
    if (!ctx || !dev_ptr || !handle)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_ipc_export: NULL argument");
    static_assert(sizeof(cudaIpcMemHandle_t) == REGK_IPC_HANDLE_BYTES, "IPC handle size");
    CK(cudaSetDevice(ctx->device));
    cudaIpcMemHandle_t h;
    CK(cudaIpcGetMemHandle(&h, const_cast<void *>(dev_ptr)));
    memcpy(handle, &h, sizeof h);
    return REGK_OK;
}

int regk_ipc_open(regk_ctx *ctx, const unsigned char handle[REGK_IPC_HANDLE_BYTES], void **peer_ptr)
{
    if (!ctx || !handle || !peer_ptr)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_ipc_open: NULL argument");
    CK(cudaSetDevice(ctx->device));
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, sizeof h);
    *peer_ptr = nullptr;
    CK(cudaIpcOpenMemHandle(peer_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return REGK_OK;
}

int regk_ipc_close(regk_ctx *ctx, void *peer_ptr)
{
    if (!ctx || !peer_ptr)
        return REGK_ERR_INVALID_ARG;
    CK(cudaSetDevice(ctx->device));
    CK(cudaIpcCloseMemHandle(peer_ptr));
    return REGK_OK;
}

int regk_gather_push(regk_ctx *ctx, const regk_result *shard, const regk_gather *g)
{
    if (!ctx || !shard || !g)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_gather_push: NULL argument");
    if (g->world == 0 || g->world > REGK_MAX_PEERS || g->rank >= g->world)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_gather_push: world %u / rank %u out of range (at most %d peers)",
            g->world, g->rank, REGK_MAX_PEERS);
    if (!(shard->flags & REGK_OUT_DEVICE) || !shard->path_off || !shard->json_off)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_gather_push: the shard must be a finished REGK_OUT_DEVICE result");
    if (!g->totals || g->rec_base + shard->n > g->n_total)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_gather_push: totals missing or record range outside the job");
    for (uint32_t q = 0; q < g->world; q++)
        if (!g->path_bytes[q] || !g->path_off[q] || !g->json_bytes[q] || !g->json_off[q] ||
            (((uintptr_t)g->path_bytes[q] | (uintptr_t)g->json_bytes[q]) & 15) || (((uintptr_t)g->path_off[q] | (uintptr_t)g->json_off[q]) & 7))
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_gather_push: buffer of rank %u missing or misaligned", q);
    CK(cudaSetDevice(ctx->device));
    if (!ctx->h_gather_flag) {
        CK(cudaMallocHost((void **)&ctx->h_gather_flag, sizeof(uint32_t)));
        *ctx->h_gather_flag = 0;
    }
    GatherParams p{};
    p.world = g->world;
    p.rank = g->rank;
    p.n_local = shard->n;
    p.rec_base = g->rec_base;
    p.n_total = g->n_total;
    p.totals = (const unsigned long long *)g->totals;
    p.src_path = shard->path_bytes;
    p.src_json = shard->json_bytes;
    p.src_path_off = (const unsigned long long *)shard->path_off;
    p.src_json_off = (const unsigned long long *)shard->json_off;
    for (uint32_t q = 0; q < g->world; q++) {
        p.dst_path[q] = (uint8_t *)g->path_bytes[q];
        p.dst_json[q] = (uint8_t *)g->json_bytes[q];
        p.dst_path_off[q] = (unsigned long long *)g->path_off[q];
        p.dst_json_off[q] = (unsigned long long *)g->json_off[q];
    }
    p.path_cap = g->path_cap;
    p.json_cap = g->json_cap;
    p.my_path_total = shard->path_total;
    p.my_json_total = shard->json_total;
    p.flag = ctx->h_gather_flag;
    regk_gather_push_kernel<<<(unsigned)ctx->sm_count * 8, 256, 0, ctx->stream>>>(p);
    CK(cudaGetLastError());
    return REGK_OK;
}

int regk_job_bind(regk_ctx *ctx, const regk_job *job)
{
    if (!ctx)
        return REGK_ERR_INVALID_ARG;
    if (ctx->pending)
        return fail(ctx, REGK_ERR_STATE, "regk_job_bind: a batch is still pending; call regk_finish first");
    if (!job) {
        ctx->job_bound = false;
        return REGK_OK;
    }
    if (job->world == 0 || job->world > REGK_MAX_PEERS || job->rank >= job->world)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_job_bind: world %u / rank %u out of range (at most %d ranks)", job->world,
            job->rank, REGK_MAX_PEERS);
    for (uint32_t q = 0; q < job->world; q++)
        if (!job->path_bytes[q] || !job->path_off[q] || !job->json_bytes[q] || !job->json_off[q] || !job->mailbox[q] ||
            (((uintptr_t)job->path_bytes[q] | (uintptr_t)job->json_bytes[q]) & 15) ||
            (((uintptr_t)job->path_off[q] | (uintptr_t)job->json_off[q] | (uintptr_t)job->mailbox[q]) & 7))
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_job_bind: buffer of rank %u missing or misaligned", q);
    CK(cudaSetDevice(ctx->device));
    int rc = ensure_dev(ctx, ctx->job_bases, (size_t)regk_ctx::NSLOTS * 64);
    if (rc)
        return rc;
    if (!ctx->h_job_bases)
        CK(cudaMallocHost((void **)&ctx->h_job_bases, (size_t)regk_ctx::NSLOTS * 64));
    if (!ctx->h_gather_flag) {
        CK(cudaMallocHost((void **)&ctx->h_gather_flag, sizeof(uint32_t)));
        *ctx->h_gather_flag = 0;
    }
    ctx->job = *job;
    ctx->job_bound = true;
    return REGK_OK;
}

/* one exchange of a job step on the context's stream (regk_peersync.cuh) */
static int launch_exchange(regk_ctx *ctx, unsigned long long v0, unsigned long long v1, const unsigned long long *src0,
    uint32_t n0, unsigned long long *bases, unsigned long long *close0)
{
    const regk_job &j = ctx->job;
    ExchangeParams e{};
    e.world = j.world;
    e.rank = j.rank;
    e.seq = ++ctx->job_seq;
    for (uint32_t q = 0; q < j.world; q++)
        e.mailbox[q] = (unsigned long long *)j.mailbox[q];
    e.v0 = v0;
    e.v1 = v1;
    e.src0 = src0;
    e.n0 = n0;
    e.bases = bases;
    e.close0 = close0;
    e.close1 = nullptr;
    e.host_flag = ctx->h_gather_flag;
    e.timeout_ns = (j.timeout_ms ? j.timeout_ms : 10000ull) * 1000000ull;
    regk_peer_exchange_kernel<<<1, 32, 0, ctx->stream>>>(e);
    CK(cudaGetLastError());
    return REGK_OK;
}

static void fill_peers(PeerDst &pd, const regk_job &j, void *const *bytes, uint64_t *const *off)
{
    pd.n = 0;
    pd.job = 1;
    /* destination order rank+1, rank+2, ...: at any moment the ranks aim at different peers */
    for (uint32_t i = 1; i < j.world; i++) {
        const uint32_t q = (j.rank + i) % j.world;
        pd.bytes[pd.n] = (uint8_t *)bytes[q];
        pd.off[pd.n] = (unsigned long long *)off[q] + j.rec_base;
        pd.n++;
    }
}

static int finish_skip(regk_ctx *ctx, regk_ctx::Slot *slot, const DevStatus &first, regk_result *res);

int regk_register_batch(regk_ctx *ctx, const regk_batch *b, regk_result *res)
{
    if (!ctx || !b || !res)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_register_batch: NULL argument");
    const bool async = opt_get(ctx, "async", 0) != 0;
    if (ctx->pending && !async)
        return fail(ctx, REGK_ERR_STATE, "regk_register_batch: previous batch not finished (regk_finish)");
    regk_ctx::Slot &slot = ctx->slots[ctx->seq % regk_ctx::NSLOTS];
    if (slot.in_use)
        return fail(ctx, REGK_ERR_STATE, "regk_register_batch: %d batches in flight; call regk_finish", regk_ctx::NSLOTS);
    memset(res, 0, sizeof *res);
    const uint64_t n = b->n;
    const bool in_dev = b->flags & REGK_IN_DEVICE;
    const bool out_dev = b->flags & REGK_OUT_DEVICE;
    const bool alias = b->flags & REGK_NODE_ALIAS;
    const bool do_path = !(b->flags & REGK_NO_PATH);
    const bool do_json = !(b->flags & REGK_NO_JSON);
    const bool job = b->flags & REGK_JOB_STEP;
    if (n >= (1ull << 32))
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_register_batch: n must be < 2^32 per call");
    if (job) {
        if (b->flags & REGK_SKIP_BAD)
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_register_batch: REGK_SKIP_BAD does not combine with REGK_JOB_STEP");
        if (!ctx->job_bound)
            return fail(ctx, REGK_ERR_STATE, "regk_register_batch: REGK_JOB_STEP without a bound job (regk_job_bind)");
        if (!in_dev || !out_dev || !do_path || !do_json)
            return fail(ctx, REGK_ERR_INVALID_ARG,
                "regk_register_batch: a job step is device-resident (REGK_IN_DEVICE | REGK_OUT_DEVICE) and produces paths and payloads");
        if (ctx->job.rec_base + n > ctx->job.n_total)
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_register_batch: the shard's record range lies outside the job");
        }
    if (do_json && ctx->types.empty())
        return fail(ctx, REGK_ERR_STATE, "regk_register_batch: call regk_set_types first");
    if (n && do_path && (!b->domain_off || (!b->domain_bytes && b->domain_bytes_len)))
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_register_batch: domain arrays missing");
    if (n && do_path && !alias && !b->host_off && b->host_stride == 0)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_register_batch: host_off is NULL and host_stride is 0");
    if (n && do_path && !alias && !b->host_bytes)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_register_batch: host_bytes missing");
    if (n && do_json && (!b->type_id || !b->addr_off))
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_register_batch: type_id / addr_off missing");
    if (n && do_json && b->ports_off && !b->ports && b->ports_len)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_register_batch: ports missing");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;

    /* ---- sizes of the packed arrays ---- */
    uint64_t dom_len = b->domain_bytes_len, host_len = b->host_bytes_len, addr_len = b->addr_bytes_len,
             ports_len = b->ports_len;
    if (!in_dev && n) {
        if (do_path) {
            dom_len = b->domain_off[n];
            host_len = alias ? 0 : (b->host_off ? b->host_off[n] : n * (uint64_t)b->host_stride);
        }
        if (do_json) {
            addr_len = b->addr_off[n];
            ports_len = b->ports_off ? b->ports_off[n] : 0;
        }
    } else if (in_dev && n) {
        if (do_path && !alias && !b->host_off)
            host_len = n * (uint64_t)b->host_stride;
        if (do_path && dom_len == 0 && b->domain_bytes)
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_register_batch: domain_bytes_len is required for device batches");
        if (do_json && addr_len == 0 && b->addr_bytes)
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_register_batch: addr_bytes_len is required for device batches");
    }
    if (alias)
        host_len = 0;

    /* Host buffers in and out, large batch: overlap H2D, kernels and D2H chunk by chunk (run_pipelined). */
    const uint64_t chunk_records = (uint64_t)opt_get(ctx, "chunk_records", 262144) / TILE * TILE;
    const bool pipelined = !in_dev && !out_dev && !async && chunk_records && n >= 2 * chunk_records &&
        !opt_get(ctx, "force_generic", 0) && chunk_bounds_ok(b, chunk_records, do_path, do_json, alias);
    /* Host buffers in and out with the "async" option: two batches may be in flight, each in its own HostSet. */
    regk_ctx::HostSet *hs = (!in_dev && !out_dev && async && n) ? &ctx->hset[ctx->hseq & 1] : nullptr;
    if (hs) {
        for (const auto &sl : ctx->slots)
            if (sl.in_use && sl.hset == (int)(ctx->hseq & 1))
                return fail(ctx, REGK_ERR_STATE,
                    "regk_register_batch: at most two host batches may be in flight; call regk_finish on the older one");
        if (!ctx->s_h2d) {
            CK(cudaStreamCreateWithFlags(&ctx->s_h2d, cudaStreamNonBlocking));
            CK(cudaStreamCreateWithFlags(&ctx->s_d2h, cudaStreamNonBlocking));
        }
        if (!hs->e_in) {
            CK(cudaEventCreateWithFlags(&hs->e_in, cudaEventDisableTiming));
            CK(cudaEventCreateWithFlags(&hs->e_out, cudaEventDisableTiming));
        }
    }
    DevBuf *stage = hs ? hs->in : ctx->in;
    DevBuf &o_path_bytes = hs ? hs->path_bytes : ctx->path_bytes, &o_path_off = hs ? hs->path_off : ctx->path_off,
           &o_json_bytes = hs ? hs->json_bytes : ctx->json_bytes, &o_json_off = hs ? hs->json_off : ctx->json_off;

    /* ---- inputs on the device ---- */
    const void *src[11] = {b->domain_bytes, b->domain_off, b->host_bytes, b->host_off, b->type_id, b->addr_bytes,
        b->addr_off, b->ttl, b->ports_off, b->ports, b->ports_present};
    const size_t sz[11] = {(size_t)dom_len, (size_t)(n + 1) * 4, (size_t)host_len, (size_t)(n + 1) * 4, (size_t)n,
        (size_t)addr_len, (size_t)(n + 1) * 4, (size_t)n * 4, (size_t)(n + 1) * 4, (size_t)ports_len * 4, (size_t)n};
    const bool need[11] = {do_path, do_path, do_path && !alias, do_path && !alias, do_json, do_json, do_json, do_json,
        do_json, do_json, do_json};
    const void *dev[11];
    for (int i = 0; i < 11; i++) {
        dev[i] = nullptr;
        if (!src[i] || !need[i] || n == 0)
            continue;
        if (in_dev) {
            if (((uintptr_t)src[i] & 15) != 0)
                return fail(ctx, REGK_ERR_INVALID_ARG, "regk_register_batch: device array %d is not 16-byte aligned", i);
            dev[i] = src[i];
        } else {
            int rc = ensure_dev(ctx, stage[i], sz[i] + 16);
            if (rc)
                return rc;
            if (sz[i] && !pipelined)
                CK(cudaMemcpyAsync(stage[i].p, src[i], sz[i], cudaMemcpyHostToDevice, hs ? ctx->s_h2d : s));
            dev[i] = stage[i].p;
        }
    }
    if (hs) {
        /* this set's staging was last read by the kernels of the batch two submissions back, which has been
           finished (checked above); the kernels below wait for the copies */
        CK(cudaEventRecord(hs->e_in, ctx->s_h2d));
        CK(cudaStreamWaitEvent(s, hs->e_in, 0));
    }

    /* ---- outputs (capacity = exact upper bounds, see DESIGN.md) ---- */
    const uint64_t path_cap = do_path ? dom_len + host_len + 2 * n + 16 : 16;
    const uint64_t json_cap = do_json ? n * (uint64_t)(38 + 2 * ctx->max_type_q + 4 + 18 + 11) + 2 * addr_len +
        11 * ports_len + 16 : 16;
    int rc;
    if (!job && ((rc = ensure_dev(ctx, o_path_bytes, path_cap)) || (rc = ensure_dev(ctx, o_path_off, (n + 1) * 8)) ||
        (rc = ensure_dev(ctx, o_json_bytes, json_cap)) || (rc = ensure_dev(ctx, o_json_off, (n + 1) * 8))))
        return rc;
    /* job step: the outputs are the rank's own whole-job buffers, every position job-absolute */
    const regk_job &J = ctx->job;
    uint8_t *const out_path_bytes = job ? (uint8_t *)J.path_bytes[J.rank] : (uint8_t *)o_path_bytes.p;
    unsigned long long *const out_path_off = job ? (unsigned long long *)J.path_off[J.rank] + J.rec_base : (unsigned long long *)o_path_off.p;
    uint8_t *const out_json_bytes = job ? (uint8_t *)J.json_bytes[J.rank] : (uint8_t *)o_json_bytes.p;
    unsigned long long *const out_json_off = job ? (unsigned long long *)J.json_off[J.rank] + J.rec_base : (unsigned long long *)o_json_off.p;
    const uint64_t out_path_cap = job ? J.path_cap : path_cap, out_json_cap = job ? J.json_cap : json_cap;
    unsigned long long *const d_bases = job ? (unsigned long long *)ctx->job_bases.p + 8 * (ctx->seq % regk_ctx::NSLOTS) : nullptr;

    /* ---- workspace: status | running payload totals per chunk | two-level byte totals of both halves ---- */
    const uint64_t ntiles = (n + TILE - 1) / TILE;
    const uint64_t nchunks = pipelined ? (n + chunk_records - 1) / chunk_records : 1;
    const uint64_t tiles_per_chunk = pipelined ? chunk_records / TILE : ntiles;
    const uint64_t nsuper_chunk = tiles_per_chunk / SUPER + 1;
    const size_t running_off = 128;
    const size_t totals_p_off = (running_off + (nchunks + 1) * 8 + 15) & ~(size_t)15;
    const size_t super_p_off = (totals_p_off + ntiles * 4 + 15) & ~(size_t)15;
    const size_t totals_j_off = super_p_off + nchunks * nsuper_chunk * 8;
    const size_t super_j_off = (totals_j_off + ntiles * 4 + 15) & ~(size_t)15;
    const size_t work_bytes = super_j_off + nchunks * nsuper_chunk * 8 + 64;
    uint8_t *wk;
    int ring = -1;
    if (pipelined) {
        if ((rc = ensure_dev(ctx, ctx->work, work_bytes)))
            return rc;
        wk = (uint8_t *)ctx->work.p;
        CK(cudaMemsetAsync(wk, 0, work_bytes, s));
    } else {
        ring = (int)(ctx->ws_seq++ % regk_ctx::NWORK);
        if (!ctx->s_side) {
            CK(cudaStreamCreateWithFlags(&ctx->s_side, cudaStreamNonBlocking));
            for (auto &e : ctx->ws_clean)
                CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        }
        const size_t cap_before = ctx->work_ring[ring].cap;
        if ((rc = ensure_dev(ctx, ctx->work_ring[ring], work_bytes)))
            return rc;
        if (ctx->work_ring[ring].cap != cap_before)
            ctx->ws_clean_bytes[ring] = 0;                  /* reallocated: contents unknown */
        wk = (uint8_t *)ctx->work_ring[ring].p;
        if (ctx->ws_clean_bytes[ring] >= work_bytes)
        {
            /* zeroed by the side stream after its last use, normally long ago: only a cleaning still in
               flight becomes a stream dependency (every extra stream operation opens a gap between kernels) */
            if (cudaEventQuery(ctx->ws_clean[ring]) != cudaSuccess) {
                cudaGetLastError();
                CK(cudaStreamWaitEvent(s, ctx->ws_clean[ring], 0));
            }
        }
        else
            CK(cudaMemsetAsync(wk, 0, work_bytes, s));
    }
    DevStatus *d_status = (DevStatus *)wk;

    if (n == 0 && !job) {
        CK(cudaMemsetAsync(o_path_off.p, 0, 8, s));
        CK(cudaMemsetAsync(o_json_off.p, 0, 8, s));
    }
    const uint32_t force_generic = (uint32_t)opt_get(ctx, "force_generic", 0);

    /* ---- kernel parameters for the whole batch ---- */
    PathParams pp{};
    size_t path_smem = 0;
    if (n && do_path) {
        pp.n = n;
        pp.domain_bytes = (const uint8_t *)dev[0];
        pp.domain_off = (const uint32_t *)dev[1];
        pp.host_bytes = (const uint8_t *)dev[2];
        pp.host_off = (const uint32_t *)dev[3];
        pp.host_stride = b->host_stride;
        pp.out_bytes = out_path_bytes;
        pp.out_off = out_path_off;
        pp.out_capacity = out_path_cap;
        if (job) {
            pp.bias_in = d_bases;
            fill_peers(pp.peer, J, J.path_bytes, J.path_off);
        }
        pp.exact = 0;                           /* closed-form offsets; see regk_finish for the exact redo */
        pp.tile_total = (uint32_t *)(wk + totals_p_off);
        pp.super_total = (unsigned long long *)(wk + super_p_off);
        pp.status = d_status;
        pp.dom_limit = dom_len;
        pp.host_limit = host_len;
        pp.force_generic = force_generic;
        /* shared-memory budget: 1.25x the mean tile, clamped; tiles that do not fit go generic */
        const uint64_t mean_dom_tile = std::min<uint64_t>(dom_len, dom_len * TILE / std::max<uint64_t>(n, 1)) + 1;  /* a FULL tile's share */
        uint32_t dom_cap = (uint32_t)opt_get(ctx, "dom_cap", 0);
        if (!dom_cap)
            dom_cap = (uint32_t)std::min<uint64_t>(std::max<uint64_t>(align16(mean_dom_tile * 5 / 4 + 384), 2048), 49152);
        dom_cap = (uint32_t)((dom_cap + 127) & ~127u);         /* bitmap region stays 16-byte aligned */
        uint32_t host_cap = 0;
        if (!alias) {
            const uint64_t mean_host_tile = pp.host_off ? std::min<uint64_t>(host_len, host_len * TILE / std::max<uint64_t>(n, 1)) + 1
                                                        : (uint64_t)TILE * b->host_stride;
            host_cap = (uint32_t)std::min<uint64_t>(align16((pp.host_off ? mean_host_tile * 3 / 2 + 512 : mean_host_tile) + 16), 49152);
        }
        const uint32_t out_cap = (uint32_t)align16((uint64_t)dom_cap + host_cap + 2 * TILE + 32);
        path_smem = 16 + (size_t)dom_cap + 32 + dom_cap / 8 + 16 + (alias ? 0 : host_cap + 32) + out_cap + 32;
        if (path_smem > (size_t)ctx->max_smem_optin)
            return fail(ctx, REGK_ERR_INVALID_ARG, "path kernel needs %zu B of shared memory (> %d)", path_smem, ctx->max_smem_optin);
        pp.dom_cap = dom_cap;
        pp.host_cap = host_cap;
        pp.out_cap = out_cap;
        if (smem_attr_needs_raise(ctx->device, alias ? 0 : 1, path_smem)) {    /* not free: only when it grows */
            if (alias) {
                CK(cudaFuncSetAttribute(regk_path_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)path_smem));
                CK(cudaFuncSetAttribute(regk_path_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)path_smem));
            } else {
                CK(cudaFuncSetAttribute(regk_path_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)path_smem));
                CK(cudaFuncSetAttribute(regk_path_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)path_smem));
            }
        }
        if ((rc = lookahead_tiles(ctx, alias ? 0 : 1, alias ? (const void *)regk_path_kernel<true, false> : (const void *)regk_path_kernel<false, false>,
                 path_smem, &pp.lookahead)))
            return rc;
    }
    JsonParams jp{};
    size_t json_smem = 0;
    if (n && do_json) {
        jp.n = n;
        jp.type_id = (const uint8_t *)dev[4];
        jp.addr_bytes = (const uint8_t *)dev[5];
        jp.addr_off = (const uint32_t *)dev[6];
        jp.ttl = (const int32_t *)dev[7];
        jp.ports_off = (const uint32_t *)dev[8];
        jp.ports = (const uint32_t *)dev[9];
        jp.ports_present = (const uint8_t *)dev[10];
        jp.frag_blob = (const uint8_t *)ctx->blob_dev.p;
        jp.ntypes = (uint32_t)ctx->types.size();
        jp.blob_bytes = (uint32_t)ctx->blob_host.size();
        jp.out_bytes = out_json_bytes;
        jp.out_off = out_json_off;
        jp.out_capacity = out_json_cap;
        if (job) {
            jp.base_in = d_bases + 4;
            fill_peers(jp.peer, J, J.json_bytes, J.json_off);
        }
        jp.tile_total = (uint32_t *)(wk + totals_j_off);
        jp.super_total = (unsigned long long *)(wk + super_j_off);
        jp.status = d_status;
        jp.addr_limit = addr_len;
        jp.ports_limit = ports_len;
        jp.force_generic = force_generic;
        uint32_t out_cap = (uint32_t)opt_get(ctx, "json_out_cap", 0);
        if (!out_cap) {
            /* mean payload estimate: fixed keys + type twice + address twice + ttl + ports - an upper estimate (the
               longest type name, six bytes per port).  Once a batch with this type table has been finished the measured
               bytes per record take over (records of one deployment look alike from batch to batch): config 3's image
               shrinks from 19.2 to 16.5 KB and two more CTAs fit an SM (payload kernel -4 %).  A budget that turns
               out too small only sends tiles down the global-memory path (counted in generic_tiles), never wrong. */
            uint64_t mean = 42 + 2ull * ctx->max_type_q + (n ? 2 * addr_len / n : 0) + 11 +
                (ports_len ? 11 + (n ? 6 * ports_len / n : 0) : 0) + 2;
            uint64_t tile_bytes = mean * TILE * 9 / 8 + 512;
            slot.json_est = mean;
            slot.json_learned = false;
            /* only for a batch that LOOKS like the one the figure was measured on (same a-priori estimate, i.e. the
               same address and port bytes per record); a learned budget that ever produced generic tiles is dropped
               for good (regk_finish) */
            if (ctx->json_mean_seen > 0.0 && n >= 4096 && ctx->json_est_seen == mean) {
                const uint64_t seen = (uint64_t)(ctx->json_mean_seen + 1.0);
                if (seen < mean) {
                    tile_bytes = seen * TILE * 17 / 16 + 1024;      /* +6 % and 1 KB: > 4.5 sigma of a 128-record sum */
                    slot.json_learned = true;
                }
            }
            out_cap = (uint32_t)std::min<uint64_t>(align16(tile_bytes), 98304);
        }
        out_cap = (uint32_t)align16(out_cap);
        jp.out_cap = out_cap;
        json_smem = (size_t)jp.blob_bytes + out_cap + 32;
        if (json_smem > (size_t)ctx->max_smem_optin)
            return fail(ctx, REGK_ERR_INVALID_ARG, "json kernel needs %zu B of shared memory (> %d)", json_smem, ctx->max_smem_optin);
        if (smem_attr_needs_raise(ctx->device, 2, json_smem)) {
            CK(cudaFuncSetAttribute(regk_json_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)json_smem));
        }
        if ((rc = lookahead_tiles(ctx, 2, (const void *)regk_json_kernel, json_smem, &jp.lookahead)))
            return rc;
    }

    if (pipelined) {
        HostPipe hp;
        hp.chunk = chunk_records;
        hp.nchunks = nchunks;
        hp.nsuper_chunk = nsuper_chunk;
        hp.running = (unsigned long long *)(wk + running_off);
        hp.path_cap = path_cap;
        hp.json_cap = json_cap;
        for (int i = 0; i < 11; i++) {
            hp.src[i] = src[i];
            hp.dev[i] = need[i] && src[i] ? ctx->in[i].p : nullptr;
        }
        rc = run_pipelined(ctx, b, res, pp, path_smem, jp, json_smem, hp);
        ctx->skip_last = regk_ctx::SkipLast{};
        if (rc == REGK_ERR_OUT_OF_DOMAIN && (b->flags & REGK_SKIP_BAD) && !(res->bad_bits & REGK_BAD_TOO_LARGE)) {
            /* the whole batch is staged in ctx->in: redo it from there like a dirty batch in regk_finish */
            slot.n = n;
            slot.flags = b->flags;
            slot.hset = -1;
            slot.off32 = false;                 /* the pipelined route returns 64-bit offsets */
            slot.timed = false;
            slot.launches = res->launches;
            for (int i = 0; i < 11; i++)
                slot.dev_in[i] = dev[i];
            slot.in_len[0] = dom_len, slot.in_len[1] = host_len, slot.in_len[2] = addr_len, slot.in_len[3] = ports_len;
            slot.in_stride = b->host_stride;
            DevStatus st{};
            st.bad_bits = res->bad_bits;
            st.first_bad = ~(unsigned long long)res->first_bad;
            return finish_skip(ctx, &slot, st, res);
        }
        if (rc == REGK_OK && (b->flags & REGK_SKIP_BAD)) {
            ctx->skip_last.valid = true;
            ctx->skip_last.n = n;
        }
        if (rc == REGK_OK) {
            ctx->last_gen++;
            ctx->last_path_bytes = do_path ? pp.out_bytes : nullptr;
            ctx->last_path_off = do_path ? pp.out_off : nullptr;
            ctx->last_n = do_path ? n : 0;
            ctx->last_json_bytes = do_json ? jp.out_bytes : nullptr;
            ctx->last_json_off = do_json ? jp.out_off : nullptr;
            ctx->last_json_n = do_json ? n : 0;
            ctx->last_host_off = pp.host_off;
            ctx->last_host_stride = pp.host_stride;
            ctx->last_alias = alias;
        }
        if (rc != REGK_ERR_STATE + 100)         /* anything but "needs the exact redo" */
            return rc;
        /* some domain has empty labels: run the whole batch again through the regular (exact-capable) path */
        for (int i = 0; i < 11; i++)
            if (dev[i] && sz[i])
                CK(cudaMemcpyAsync(ctx->in[i].p, src[i], sz[i], cudaMemcpyHostToDevice, s));
        CK(cudaMemsetAsync(wk, 0, work_bytes, s));
    }

    uint32_t launches = 0;
    slot.did_path = false;
    slot.d_status = d_status;
    slot.dev_path_bytes = (n && do_path && !job) ? pp.out_bytes : nullptr;    /* regk_parent_dirs: not on job steps */
    slot.dev_path_off = (n && do_path && !job) ? pp.out_off : nullptr;
    slot.dev_json_bytes = (n && do_json && !job) ? jp.out_bytes : nullptr;
    slot.dev_json_off = (n && do_json && !job) ? jp.out_off : nullptr;
    slot.dev_host_off = pp.host_off;
    slot.host_stride = pp.host_stride;
    slot.alias = alias;
    const bool fused_len = n && do_path && do_json;
    /* per-kernel timing events sit between the launches and cost a few microseconds of stream gaps per batch:
       "time_every" = K keeps them on every K-th batch only (the others report kernel times of 0) */
    const int64_t time_every = std::max<int64_t>(1, opt_get(ctx, "time_every", 1));
    const bool timed = ctx->seq % (uint64_t)time_every == 0;
    slot.timed = timed;
    if (job) {
        /* exchange 1 (entry barrier): closed-form path bytes of every shard -> this rank's path base; the job's
           closing path offset lands in this rank's own offset array */
        const uint64_t my_paths = dom_len + host_len + (alias ? 1 : 2) * n;
        if ((rc = launch_exchange(ctx, my_paths, n, nullptr, 0, d_bases, (unsigned long long *)J.path_off[J.rank] + J.n_total)))
            return rc;
        launches++;
    }
    if (timed)
        CK(cudaEventRecord(slot.ev[0], s));
    if (n && do_path) {
        if (alias)
            regk_path_kernel<true, false><<<(unsigned)ntiles, TILE, path_smem, s>>>(pp, fused_len ? jp : JsonParams{});
        else
            regk_path_kernel<false, false><<<(unsigned)ntiles, TILE, path_smem, s>>>(pp, fused_len ? jp : JsonParams{});
        CK(cudaGetLastError());
        launches++;
        slot.path_params = pp;
        slot.path_smem = path_smem;
        slot.path_alias = alias;
        slot.did_path = true;
    }
    if (timed)
        CK(cudaEventRecord(slot.ev[1], s));
    if (job) {
        /* exchange 2: payload bytes of every shard (sum of the super-tile totals the path kernel's side job left)
           -> this rank's payload base */
        if ((rc = launch_exchange(ctx, 0, 0, n ? jp.super_total : nullptr, n ? (uint32_t)nsuper_chunk : 0, d_bases + 4,
                 (unsigned long long *)J.json_off[J.rank] + J.n_total)))
            return rc;
        launches++;
    }
    if (n && do_json) {
        if (!fused_len) {
            const unsigned len_grid = (unsigned)std::min<uint64_t>(ntiles, (uint64_t)ctx->sm_count * 8);
            regk_json_len_kernel<<<len_grid, TILE, 0, s>>>(jp, (uint32_t)ntiles);
            CK(cudaGetLastError());
            launches++;
        }
        if (timed)
            CK(cudaEventRecord(slot.ev[2], s));
        regk_json_kernel<<<(unsigned)ntiles, TILE, json_smem, s>>>(jp);
        CK(cudaGetLastError());
        launches++;
    } else if (timed) {
        CK(cudaEventRecord(slot.ev[2], s));
    }
    slot.off32 = !out_dev && !job && n && opt_get(ctx, "offsets32", 0) != 0;
    if (slot.off32) {
        if (do_path && (rc = narrow_offsets(ctx, o_path_off.p, hs ? hs->off32_p : ctx->off32_p, n, s)))
            return rc;
        if (do_json && (rc = narrow_offsets(ctx, o_json_off.p, hs ? hs->off32_j : ctx->off32_j, n, s)))
            return rc;
    }
    CK(cudaEventRecord(slot.ev[3], s));
    if (job) {
        /* exchange 3 (closing barrier): once it has passed, every rank's tiles and offsets are in this rank's buffers */
        if ((rc = launch_exchange(ctx, 0, 0, nullptr, 0, nullptr, nullptr)))
            return rc;
        launches++;
        CK(cudaEventRecord(slot.ev[5], s));
    }
    if (ring >= 0) {
        /* off the main stream: status read-back, then re-zero this workspace for its next turn */
        CK(cudaStreamWaitEvent(ctx->s_side, job ? slot.ev[5] : slot.ev[3], 0));
        CK(cudaMemcpyAsync(slot.h_status, d_status, sizeof(DevStatus), cudaMemcpyDeviceToHost, ctx->s_side));
        if (job)
            CK(cudaMemcpyAsync(ctx->h_job_bases + 8 * (ctx->seq % regk_ctx::NSLOTS), d_bases, 64, cudaMemcpyDeviceToHost, ctx->s_side));
        CK(cudaEventRecord(slot.ev[4], ctx->s_side));
        CK(cudaMemsetAsync(wk, 0, work_bytes, ctx->s_side));
        CK(cudaEventRecord(ctx->ws_clean[ring], ctx->s_side));
        ctx->ws_clean_bytes[ring] = work_bytes;
        slot.ring = ring;
    } else {
        CK(cudaMemcpyAsync(slot.h_status, d_status, sizeof(DevStatus), cudaMemcpyDeviceToHost, s));
        CK(cudaEventRecord(slot.ev[4], s));
        slot.ring = -1;
    }

    slot.hset = hs ? (int)(hs - ctx->hset) : -1;
    slot.job = job;
    slot.d2h_issued = false;
    slot.in_use = true;
    slot.n = n;
    slot.flags = b->flags;
    slot.launches = launches;
    for (int i = 0; i < 11; i++)
        slot.dev_in[i] = dev[i];
    slot.in_len[0] = dom_len, slot.in_len[1] = host_len, slot.in_len[2] = addr_len, slot.in_len[3] = ports_len;
    slot.in_stride = b->host_stride;
    ctx->seq++;
    ctx->pending++;
    res->n = n;
    res->flags = out_dev ? REGK_OUT_DEVICE : 0;
    res->launches = launches;
    res->opaque = &slot;
    if (hs) {
        /* the other set's batch, if still open: its kernels ran ahead of this batch's copies - start its D2H now
           so that it overlaps this batch's H2D */
        ctx->hseq++;
        for (auto &sl : ctx->slots)
            if (&sl != &slot && sl.in_use && sl.hset >= 0 && !sl.d2h_issued) {
                cudaError_t e = cudaEventSynchronize(sl.ev[4]);
                if (e != cudaSuccess)
                    return fail(ctx, REGK_ERR_CUDA, "kernel execution failed: %s", cudaGetErrorString(e));
                if ((rc = issue_d2h(ctx, sl)))
                    return rc;
            }
    }
    if (async)
        return REGK_OK;
    return regk_finish(ctx, res);
}

/*
 * Skip mode, dirty batch (regk_skip.cuh): the first pass found out-of-domain records and no REGK_BAD_TOO_LARGE.
 * Fence pass -> compaction of the kept records into ctx->skip_in -> that batch through regk_register_batch as an
 * ordinary device batch (its outputs, in ctx->path_bytes / json_bytes, are the result's streams and what the
 * downstream calls on the batch finished last see) -> offsets expanded to all n records.  Timings describe the
 * first pass, as for the exact-offset redo; launches count every kernel of the call.
 */
static int finish_skip(regk_ctx *ctx, regk_ctx::Slot *slot, const DevStatus &first, regk_result *res)
{
    cudaStream_t s = ctx->stream;
    const uint64_t n = slot->n;
    const uint32_t flags = slot->flags;
    const bool alias = flags & REGK_NODE_ALIAS, do_path = !(flags & REGK_NO_PATH), do_json = !(flags & REGK_NO_JSON);
    const bool out_dev = flags & REGK_OUT_DEVICE;
    if (ctx->pending) {
        /* the redo writes the device outputs and reads this batch's inputs: only other host-set batches may be open */
        bool ok = slot->hset >= 0;
        for (const auto &sl : ctx->slots)
            if (sl.in_use && sl.hset < 0)
                ok = false;
        if (!ok)
            return fail(ctx, REGK_ERR_STATE,
                "batch needs the skip-mode redo but later batches are in flight; finish them in order");
    }
    float ms_p = 0, ms_jl = 0, ms_j = 0;
    if (slot->timed) {
        cudaEventElapsedTime(&ms_p, slot->ev[0], slot->ev[1]);
        cudaEventElapsedTime(&ms_jl, slot->ev[1], slot->ev[2]);
        cudaEventElapsedTime(&ms_j, slot->ev[2], slot->ev[3]);
    }
    int rc;

    /* ---- 1. fence pass: per-record bits, tile totals of the kept records ---- */
    const uint64_t ntiles = (n + TILE - 1) / TILE, nsuper = ntiles / SUPER + 1;
    const size_t tt_bytes = align16(ntiles * 4), st_bytes = nsuper * 8;
    const size_t bits_off = 128 + SKIP_Q * (tt_bytes + st_bytes);
    static_assert(sizeof(SkipStatus) <= 128, "SkipStatus");
    if ((rc = ensure_dev(ctx, ctx->skip_work, bits_off + align16(n) + 16)) || (rc = ensure_host(ctx, ctx->h_skip_status, sizeof(SkipStatus))))
        return rc;
    uint8_t *wk = (uint8_t *)ctx->skip_work.p;
    CK(cudaMemsetAsync(wk, 0, bits_off, s));
    SkipParams sp{};
    sp.n = n;
    sp.alias = alias;
    sp.do_path = do_path;
    sp.do_json = do_json;
    sp.ntypes = (uint32_t)ctx->types.size();
    sp.domain_bytes = (const uint8_t *)slot->dev_in[0];
    sp.domain_off = (const uint32_t *)slot->dev_in[1];
    sp.host_bytes = (const uint8_t *)slot->dev_in[2];
    sp.host_off = (const uint32_t *)slot->dev_in[3];
    sp.host_stride = slot->in_stride;
    sp.type_id = (const uint8_t *)slot->dev_in[4];
    sp.addr_bytes = (const uint8_t *)slot->dev_in[5];
    sp.addr_off = (const uint32_t *)slot->dev_in[6];
    sp.ttl = (const int32_t *)slot->dev_in[7];
    sp.ports_off = (const uint32_t *)slot->dev_in[8];
    sp.ports = (const uint32_t *)slot->dev_in[9];
    sp.ports_present = (const uint8_t *)slot->dev_in[10];
    sp.status = (SkipStatus *)wk;
    for (int j = 0; j < SKIP_Q; j++) {
        sp.tile_total[j] = (uint32_t *)(wk + 128 + j * tt_bytes);
        sp.super_total[j] = (unsigned long long *)(wk + 128 + SKIP_Q * tt_bytes + j * st_bytes);
    }
    sp.bits = wk + bits_off;
    regk_fence_kernel<<<(unsigned)ntiles, TILE, 0, s>>>(sp);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(ctx->h_skip_status.p, sp.status, sizeof(SkipStatus), cudaMemcpyDeviceToHost, s));
    cudaError_t e = cudaStreamSynchronize(s);
    if (e != cudaSuccess)
        return fail(ctx, REGK_ERR_CUDA, "skip-mode fence pass failed: %s", cudaGetErrorString(e));
    const SkipStatus fs = *(const SkipStatus *)ctx->h_skip_status.p;
    if (fs.bad_bits != first.bad_bits || fs.first_bad != first.first_bad)
        return fail(ctx, REGK_ERR_CUDA,
            "internal error: the skip-mode fence (bits 0x%x, first record %llu) disagrees with the compose kernels (0x%x, %llu)",
            fs.bad_bits, ~fs.first_bad, first.bad_bits, ~first.first_bad);

    /* ---- 2. compaction into the scratch batch ---- */
    const uint64_t kept = fs.total[SKIP_REC], nskip = n - kept;
    const uint64_t c_dom = fs.total[SKIP_DOM], c_addr = fs.total[SKIP_ADDR], c_ports = fs.total[SKIP_PORTS];
    const uint64_t c_host = (!do_path || alias) ? 0 : (sp.host_off ? fs.total[SKIP_HOST] : kept * (uint64_t)sp.host_stride);
    const size_t csz[11] = {(size_t)c_dom, (size_t)(kept + 1) * 4, (size_t)c_host, (size_t)(kept + 1) * 4, (size_t)kept,
        (size_t)c_addr, (size_t)(kept + 1) * 4, (size_t)kept * 4, (size_t)(kept + 1) * 4, (size_t)c_ports * 4, (size_t)kept};
    void *cin[11];
    for (int i = 0; i < 11; i++) {
        cin[i] = nullptr;
        if (!slot->dev_in[i])
            continue;
        if ((rc = ensure_dev(ctx, ctx->skip_in[i], csz[i] + 16)))
            return rc;
        cin[i] = ctx->skip_in[i].p;
    }
    if ((rc = ensure_dev(ctx, ctx->skip_index, nskip * 8 + 16)) || (rc = ensure_dev(ctx, ctx->skip_bits, nskip + 16)))
        return rc;
    sp.c_domain_bytes = (uint8_t *)cin[0];
    sp.c_domain_off = (uint32_t *)cin[1];
    sp.c_host_bytes = (uint8_t *)cin[2];
    sp.c_host_off = (uint32_t *)cin[3];
    sp.c_type_id = (uint8_t *)cin[4];
    sp.c_addr_bytes = (uint8_t *)cin[5];
    sp.c_addr_off = (uint32_t *)cin[6];
    sp.c_ttl = (int32_t *)cin[7];
    sp.c_ports_off = (uint32_t *)cin[8];
    sp.c_ports = (uint32_t *)cin[9];
    sp.c_ports_present = (uint8_t *)cin[10];
    sp.skip_index = (unsigned long long *)ctx->skip_index.p;
    sp.skip_bits = (uint8_t *)ctx->skip_bits.p;
    regk_compact_kernel<<<(unsigned)ntiles, TILE, 0, s>>>(sp);
    CK(cudaGetLastError());

    /* ---- the kept records alone, as an ordinary device batch (exact-offset redo included) ---- */
    regk_batch cb{};
    cb.n = kept;
    cb.flags = REGK_IN_DEVICE | REGK_OUT_DEVICE | (flags & (REGK_NODE_ALIAS | REGK_NO_JSON | REGK_NO_PATH));
    cb.host_stride = slot->in_stride;
    cb.domain_bytes_len = c_dom;
    cb.host_bytes_len = c_host;
    cb.addr_bytes_len = c_addr;
    cb.ports_len = c_ports;
    cb.domain_bytes = c_dom ? (const uint8_t *)cin[0] : nullptr;    /* a device batch declares a non-empty array's length */
    cb.domain_off = (const uint32_t *)cin[1];
    cb.host_bytes = c_host ? (const uint8_t *)cin[2] : nullptr;
    cb.host_off = (const uint32_t *)cin[3];
    cb.type_id = (const uint8_t *)cin[4];
    cb.addr_bytes = c_addr ? (const uint8_t *)cin[5] : nullptr;
    cb.addr_off = (const uint32_t *)cin[6];
    cb.ttl = (const int32_t *)cin[7];
    cb.ports_off = (const uint32_t *)cin[8];
    cb.ports = c_ports ? (const uint32_t *)cin[9] : nullptr;
    cb.ports_present = (const uint8_t *)cin[10];
    /* synchronous, and without learning a payload budget: the second run is not a batch the caller submitted */
    const auto async_it = ctx->opt.find("async");
    const bool had_async = async_it != ctx->opt.end();
    const int64_t async_was = had_async ? async_it->second : 0;
    const int pending_was = ctx->pending;
    const double mean_was = ctx->json_mean_seen;
    const uint64_t est_was = ctx->json_est_seen;
    const bool learning_was = ctx->json_learning;
    ctx->opt["async"] = 0;
    ctx->pending = 0;
    regk_result cres;
    rc = regk_register_batch(ctx, &cb, &cres);
    if (had_async)
        ctx->opt["async"] = async_was;
    else
        ctx->opt.erase("async");
    ctx->pending = pending_was;
    ctx->json_mean_seen = mean_was;
    ctx->json_est_seen = est_was;
    ctx->json_learning = learning_was;
    if (rc == REGK_ERR_OUT_OF_DOMAIN || (rc == REGK_OK && cres.bad_bits))
        return fail(ctx, REGK_ERR_CUDA, "internal error: the kept records of a skip-mode batch still fail the fence (bits 0x%x)",
            cres.bad_bits);
    if (rc)
        return rc;

    /* ---- 3. offsets of all n records ---- */
    if ((rc = ensure_dev(ctx, ctx->skip_off_p, (n + 1) * 8)) || (rc = ensure_dev(ctx, ctx->skip_off_j, (n + 1) * 8)))
        return rc;
    ExpandParams ep{};
    ep.n = n;
    ep.bits = sp.bits;
    ep.tile_total = sp.tile_total[SKIP_REC];
    ep.super_total = sp.super_total[SKIP_REC];
    ep.c_path_off = do_path ? (const unsigned long long *)cres.path_off : nullptr;
    ep.c_json_off = do_json ? (const unsigned long long *)cres.json_off : nullptr;
    ep.path_off = (unsigned long long *)ctx->skip_off_p.p;
    ep.json_off = (unsigned long long *)ctx->skip_off_j.p;
    regk_expand_kernel<<<(unsigned)(n / TILE + 1), TILE, 0, s>>>(ep);
    CK(cudaGetLastError());
    if (!do_path)
        CK(cudaMemsetAsync(ctx->skip_off_p.p, 0, (n + 1) * 8, s));
    if (!do_json)
        CK(cudaMemsetAsync(ctx->skip_off_j.p, 0, (n + 1) * 8, s));
    uint32_t launches = slot->launches + 3 + cres.launches;
    const bool off32 = slot->off32 && !out_dev && cres.path_total < (1ull << 32) && cres.json_total < (1ull << 32);
    if (off32) {
        if ((rc = narrow_offsets(ctx, ctx->skip_off_p.p, ctx->off32_p, n, s)) || (rc = narrow_offsets(ctx, ctx->skip_off_j.p, ctx->off32_j, n, s)))
            return rc;
        launches += 2;
    }

    memset(res, 0, sizeof *res);
    res->n = n;
    res->bad_bits = first.bad_bits;
    res->first_bad = ~first.first_bad;
    res->path_total = cres.path_total;
    res->json_total = cres.json_total;
    res->path_kernel_ms = ms_p;
    res->json_kernel_ms = ms_j;
    res->json_len_kernel_ms = ms_jl;
    res->kernel_ms = ms_p + ms_jl + ms_j;
    res->launches = launches;
    res->generic_tiles = cres.generic_tiles;
    if (out_dev) {
        res->flags = REGK_OUT_DEVICE;
        res->path_bytes = cres.path_bytes;
        res->path_off = (uint64_t *)ctx->skip_off_p.p;
        res->json_bytes = cres.json_bytes;
        res->json_off = (uint64_t *)ctx->skip_off_j.p;
        e = cudaStreamSynchronize(s);
        if (e != cudaSuccess)
            return fail(ctx, REGK_ERR_CUDA, "skip-mode offset expansion failed: %s", cudaGetErrorString(e));
    } else {
        regk_ctx::HostSet *hs = slot->hset >= 0 ? &ctx->hset[slot->hset] : nullptr;
        HostBuf &hpb = hs ? hs->h_path_bytes : ctx->h_path_bytes, &hpo = hs ? hs->h_path_off : ctx->h_path_off,
                &hjb = hs ? hs->h_json_bytes : ctx->h_json_bytes, &hjo = hs ? hs->h_json_off : ctx->h_json_off;
        if ((rc = ensure_host(ctx, hpb, cres.path_total + 16)) || (rc = ensure_host(ctx, hpo, (n + 1) * 8)) ||
            (rc = ensure_host(ctx, hjb, cres.json_total + 16)) || (rc = ensure_host(ctx, hjo, (n + 1) * 8)))
            return rc;
        const size_t ow = off32 ? 4 : 8;
        if (do_path) {
            CK(cudaMemcpyAsync(hpb.p, cres.path_bytes, cres.path_total, cudaMemcpyDeviceToHost, s));
            CK(cudaMemcpyAsync(hpo.p, off32 ? ctx->off32_p.p : ctx->skip_off_p.p, (n + 1) * ow, cudaMemcpyDeviceToHost, s));
        } else {
            memset(hpo.p, 0, (n + 1) * 8);
        }
        if (do_json) {
            CK(cudaMemcpyAsync(hjb.p, cres.json_bytes, cres.json_total, cudaMemcpyDeviceToHost, s));
            CK(cudaMemcpyAsync(hjo.p, off32 ? ctx->off32_j.p : ctx->skip_off_j.p, (n + 1) * ow, cudaMemcpyDeviceToHost, s));
        } else {
            memset(hjo.p, 0, (n + 1) * 8);
        }
        e = cudaStreamSynchronize(s);
        if (e != cudaSuccess)
            return fail(ctx, REGK_ERR_CUDA, "skip-mode result copy failed: %s", cudaGetErrorString(e));
        res->flags = 0;
        res->path_bytes = (uint8_t *)hpb.p;
        res->json_bytes = (uint8_t *)hjb.p;
        if (off32) {
            res->path_off32 = (uint32_t *)hpo.p;
            res->json_off32 = (uint32_t *)hjo.p;
        } else {
            res->path_off = (uint64_t *)hpo.p;
            res->json_off = (uint64_t *)hjo.p;
        }
    }
    ctx->skip_last.valid = true;
    ctx->skip_last.n = n;
    ctx->skip_last.n_skipped = nskip;
    ctx->skip_last.bad_bits = fs.bad_bits;
    return REGK_OK;
}

int regk_skipped_records(regk_ctx *ctx, uint32_t flags, regk_skipped *out)
{
    if (!ctx || !out)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_skipped_records: NULL argument");
    if (!ctx->skip_last.valid)
        return fail(ctx, REGK_ERR_STATE, "regk_skipped_records: the batch finished last was not a REGK_SKIP_BAD batch");
    memset(out, 0, sizeof *out);
    const regk_ctx::SkipLast &sl = ctx->skip_last;
    out->n = sl.n;
    out->n_skipped = sl.n_skipped;
    out->bad_bits = sl.bad_bits;
    if (!sl.n_skipped)
        return REGK_OK;
    if (flags & REGK_OUT_DEVICE) {
        out->flags = REGK_OUT_DEVICE;
        out->index = (const uint64_t *)ctx->skip_index.p;
        out->bits = (const uint8_t *)ctx->skip_bits.p;
        return REGK_OK;
    }
    CK(cudaSetDevice(ctx->device));
    int rc;
    if ((rc = ensure_host(ctx, ctx->h_skip_index, sl.n_skipped * 8)) || (rc = ensure_host(ctx, ctx->h_skip_bits, sl.n_skipped)))
        return rc;
    CK(cudaMemcpyAsync(ctx->h_skip_index.p, ctx->skip_index.p, sl.n_skipped * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(ctx->h_skip_bits.p, ctx->skip_bits.p, sl.n_skipped, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    out->index = (const uint64_t *)ctx->h_skip_index.p;
    out->bits = (const uint8_t *)ctx->h_skip_bits.p;
    return REGK_OK;
}

int regk_finish(regk_ctx *ctx, regk_result *res)
{
    if (!ctx || !res)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_finish: NULL argument");
    regk_ctx::Slot *slot = (regk_ctx::Slot *)res->opaque;
    if (!slot || slot < ctx->slots || slot >= ctx->slots + regk_ctx::NSLOTS || !slot->in_use)
        return fail(ctx, REGK_ERR_STATE, "regk_finish: this result has no batch in flight");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    cudaError_t e = cudaEventSynchronize(slot->ev[4]);
    slot->in_use = false;
    ctx->pending--;
    if (e != cudaSuccess)
        return fail(ctx, REGK_ERR_CUDA, "kernel execution failed: %s", cudaGetErrorString(e));
    uint32_t extra_launches = 0;
    if (slot->job) {
        if (ctx->h_gather_flag && *ctx->h_gather_flag == 2u) {
            *ctx->h_gather_flag = 0;
            return fail(ctx, REGK_ERR_CUDA, "job step: a peer did not reach the exchange in time (mailbox wait timed out)");
        }
        if (slot->h_status->needs_exact && !slot->h_status->bad_bits)
            return fail(ctx, REGK_ERR_STATE,
                "job step: a domain has empty labels, so the closed-form placement of the fused all-gather does not hold; "
                "run this shard as a plain batch and reassemble with regk_gather_push");
    }
    if (!slot->job && slot->h_status->needs_exact && !slot->h_status->bad_bits && slot->did_path) {
        /* Some domain has empty labels (path.join drops them): the closed-form offsets do not hold.
           Re-run the path half with exact lengths: length kernel + last-CTA scan, then compose. */
        if (ctx->pending && slot->hset < 0)         /* device outputs are single-buffered; host sets are not */
            return fail(ctx, REGK_ERR_STATE,
                "batch needs the exact-offset redo but later batches are in flight; finish them in order");
        PathParams p = slot->path_params;
        const unsigned ntiles_r = (unsigned)((p.n + TILE - 1) / TILE);
        const unsigned long long json_total_first = slot->h_status->json_total;
        if (slot->ring >= 0) {
            CK(cudaStreamWaitEvent(s, ctx->ws_clean[slot->ring], 0));   /* the side stream has re-zeroed it: what the redo needs */
            ctx->ws_clean_bytes[slot->ring] = 0;                            /* ... and the redo dirties it again */
        }
        CK(cudaMemsetAsync(&slot->d_status->needs_exact, 0, sizeof(uint32_t), s));
        /* the path totals were zeroed with the workspace and nothing has touched them yet */
        if (slot->path_alias)
            regk_path_len_kernel<true><<<ntiles_r, TILE, 0, s>>>(p);
        else
            regk_path_len_kernel<false><<<ntiles_r, TILE, 0, s>>>(p);
        CK(cudaGetLastError());
        p.exact = 1;
        if (slot->path_alias)
            regk_path_kernel<true, true><<<ntiles_r, TILE, slot->path_smem, s>>>(p, JsonParams{});
        else
            regk_path_kernel<false, true><<<ntiles_r, TILE, slot->path_smem, s>>>(p, JsonParams{});
        CK(cudaGetLastError());
        if (slot->off32) {
            int rc2 = narrow_offsets(ctx, p.out_off, slot->hset >= 0 ? ctx->hset[slot->hset].off32_p : ctx->off32_p, p.n, s);
            if (rc2)
                return rc2;
        }
        CK(cudaMemcpyAsync(slot->h_status, slot->d_status, sizeof(DevStatus), cudaMemcpyDeviceToHost, s));
        e = cudaStreamSynchronize(s);
        if (e != cudaSuccess)
            return fail(ctx, REGK_ERR_CUDA, "exact-offset redo failed: %s", cudaGetErrorString(e));
        if (slot->ring >= 0)
            slot->h_status->json_total = json_total_first;  /* the payload half was not re-run */
        extra_launches = 2;
    }
    const DevStatus st = *slot->h_status;
    const uint64_t n = slot->n;
    const bool out_dev = slot->flags & REGK_OUT_DEVICE;
    ctx->skip_last = regk_ctx::SkipLast{};
    if (slot->flags & REGK_SKIP_BAD) {
        if (st.bad_bits && !(st.bad_bits & REGK_BAD_TOO_LARGE) && !st.overflow)
            return finish_skip(ctx, slot, st, res);
        if (!st.bad_bits) {
            ctx->skip_last.valid = true;
            ctx->skip_last.n = n;
        }
    }
    ctx->last_gen++;
    ctx->last_path_bytes = st.bad_bits ? nullptr : slot->dev_path_bytes;
    ctx->last_path_off = st.bad_bits ? nullptr : slot->dev_path_off;
    ctx->last_n = (st.bad_bits || !slot->dev_path_off) ? 0 : n;
    ctx->last_json_bytes = st.bad_bits ? nullptr : slot->dev_json_bytes;
    ctx->last_json_off = st.bad_bits ? nullptr : slot->dev_json_off;
    ctx->last_json_n = (st.bad_bits || !slot->dev_json_off) ? 0 : n;
    ctx->last_host_off = slot->dev_host_off;
    ctx->last_host_stride = slot->host_stride;
    ctx->last_alias = slot->alias;
    float ms_p = 0, ms_jl = 0, ms_j = 0;
    if (slot->timed) {
        cudaEventElapsedTime(&ms_p, slot->ev[0], slot->ev[1]);
        cudaEventElapsedTime(&ms_jl, slot->ev[1], slot->ev[2]);
        cudaEventElapsedTime(&ms_j, slot->ev[2], slot->ev[3]);
    }
    res->n = n;
    res->path_kernel_ms = ms_p;
    res->json_kernel_ms = ms_j;
    res->json_len_kernel_ms = ms_jl;
    res->kernel_ms = ms_p + ms_jl + ms_j;
    res->launches = slot->launches + extra_launches;
    res->bad_bits = st.bad_bits;
    res->first_bad = st.bad_bits ? ~st.first_bad : 0;
    res->path_total = st.path_total;
    res->json_total = st.json_total;
    res->generic_tiles = st.generic_tiles;
    if (slot->json_learned && st.generic_tiles) {
        ctx->json_learning = false;             /* the measured mean misjudged this workload once: never again */
        ctx->json_mean_seen = 0.0;
    } else if (ctx->json_learning && !st.bad_bits && !st.overflow && n >= 4096 && st.json_total && slot->json_est) {
        ctx->json_mean_seen = (double)st.json_total / (double)n;
        ctx->json_est_seen = slot->json_est;
    }
    if (st.overflow)
        return fail(ctx, REGK_ERR_CUDA, "internal error: output capacity bound exceeded");
    if (st.bad_bits) {
        res->path_total = res->json_total = 0;
        return fail(ctx, REGK_ERR_OUT_OF_DOMAIN,
            "record %llu is outside the supported input domain (REGK_BAD bits 0x%x); no output produced",
            (unsigned long long)res->first_bad, st.bad_bits);
    }
    if (slot->job) {
        const unsigned long long *hb = ctx->h_job_bases + 8 * ((size_t)(slot - ctx->slots));
        res->flags = REGK_OUT_DEVICE;
        res->path_bytes = (uint8_t *)ctx->job.path_bytes[ctx->job.rank];
        res->path_off = ctx->job.path_off[ctx->job.rank];
        res->json_bytes = (uint8_t *)ctx->job.json_bytes[ctx->job.rank];
        res->json_off = ctx->job.json_off[ctx->job.rank];
        res->job_path_base = hb[0];
        res->job_path_total = hb[1];
        res->job_json_base = hb[4];
        res->job_json_total = hb[5];
        return REGK_OK;
    }
    if (out_dev) {
        res->flags = REGK_OUT_DEVICE;
        res->path_bytes = (uint8_t *)ctx->path_bytes.p;
        res->path_off = (uint64_t *)ctx->path_off.p;
        res->json_bytes = (uint8_t *)ctx->json_bytes.p;
        res->json_off = (uint64_t *)ctx->json_off.p;
        return REGK_OK;
    }
    int rc;
    if (slot->hset >= 0) {
        regk_ctx::HostSet &hs = ctx->hset[slot->hset];
        if (!slot->d2h_issued && (rc = issue_d2h(ctx, *slot)))
            return rc;
        e = cudaEventSynchronize(hs.e_out);
        if (e != cudaSuccess)
            return fail(ctx, REGK_ERR_CUDA, "device-to-host copy failed: %s", cudaGetErrorString(e));
        res->flags = 0;
        res->path_bytes = (uint8_t *)hs.h_path_bytes.p;
        res->json_bytes = (uint8_t *)hs.h_json_bytes.p;
        if (slot->off32) {
            res->path_off32 = (uint32_t *)hs.h_path_off.p;
            res->json_off32 = (uint32_t *)hs.h_json_off.p;
        } else {
            res->path_off = (uint64_t *)hs.h_path_off.p;
            res->json_off = (uint64_t *)hs.h_json_off.p;
        }
        return REGK_OK;
    }
    const bool do_path = !(slot->flags & REGK_NO_PATH), do_json = !(slot->flags & REGK_NO_JSON);
    if ((rc = ensure_host(ctx, ctx->h_path_bytes, st.path_total + 16)) || (rc = ensure_host(ctx, ctx->h_path_off, (n + 1) * 8)) ||
        (rc = ensure_host(ctx, ctx->h_json_bytes, st.json_total + 16)) || (rc = ensure_host(ctx, ctx->h_json_off, (n + 1) * 8)))
        return rc;
    slot->off32 = slot->off32 && st.path_total < (1ull << 32) && st.json_total < (1ull << 32);
    const size_t ow = slot->off32 ? 4 : 8;
    if (n && do_path) {
        CK(cudaMemcpyAsync(ctx->h_path_bytes.p, ctx->path_bytes.p, st.path_total, cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(ctx->h_path_off.p, slot->off32 ? ctx->off32_p.p : ctx->path_off.p, (n + 1) * ow, cudaMemcpyDeviceToHost, s));
    } else {
        memset(ctx->h_path_off.p, 0, (n + 1) * 8);
    }
    if (n && do_json) {
        CK(cudaMemcpyAsync(ctx->h_json_bytes.p, ctx->json_bytes.p, st.json_total, cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(ctx->h_json_off.p, slot->off32 ? ctx->off32_j.p : ctx->json_off.p, (n + 1) * ow, cudaMemcpyDeviceToHost, s));
    } else {
        memset(ctx->h_json_off.p, 0, (n + 1) * 8);
    }
    CK(cudaStreamSynchronize(s));
    res->flags = 0;
    res->path_bytes = (uint8_t *)ctx->h_path_bytes.p;
    res->json_bytes = (uint8_t *)ctx->h_json_bytes.p;
    if (slot->off32) {
        res->path_off32 = (uint32_t *)ctx->h_path_off.p;
        res->json_off32 = (uint32_t *)ctx->h_json_off.p;
    } else {
        res->path_off = (uint64_t *)ctx->h_path_off.p;
        res->json_off = (uint64_t *)ctx->h_json_off.p;
    }
    return REGK_OK;
}

int regk_service_records(regk_ctx *ctx, const regk_service_batch *b, regk_result *res)
{
    if (!ctx || !b || !res)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_service_records: NULL argument");
    if (ctx->pending)
        return fail(ctx, REGK_ERR_STATE, "regk_service_records: batches are still in flight; finish them first");
    memset(res, 0, sizeof *res);
    const uint64_t n = b->n;
    const bool in_dev = b->flags & REGK_IN_DEVICE, out_dev = b->flags & REGK_OUT_DEVICE;
    if (n >= (1ull << 32))
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_service_records: n must be < 2^32 per call");
    if (n && (!b->srvce_off || !b->proto_off || !b->port || !b->ttl))
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_service_records: srvce_off / proto_off / port / ttl missing");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    uint64_t srvce_len = b->srvce_bytes_len, proto_len = b->proto_bytes_len;
    if (!in_dev && n) {
        srvce_len = b->srvce_off[n];
        proto_len = b->proto_off[n];
    }
    if (n && ((srvce_len && !b->srvce_bytes) || (proto_len && !b->proto_bytes)))
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_service_records: string bytes missing");
    const void *src[7] = {b->srvce_bytes, b->srvce_off, b->proto_bytes, b->proto_off, b->port, b->ttl, b->key_order};
    const size_t sz[7] = {(size_t)srvce_len, (size_t)(n + 1) * 4, (size_t)proto_len, (size_t)(n + 1) * 4, (size_t)n * 4,
        (size_t)n * 4, (size_t)n};
    const void *dev[7];
    int rc;
    for (int i = 0; i < 7; i++) {
        dev[i] = nullptr;
        if (!src[i] || n == 0)
            continue;
        if (in_dev) {
            if (((uintptr_t)src[i] & 15) != 0)
                return fail(ctx, REGK_ERR_INVALID_ARG, "regk_service_records: device array %d is not 16-byte aligned", i);
            dev[i] = src[i];
        } else {
            if ((rc = ensure_dev(ctx, ctx->svc_in[i], sz[i] + 16)))
                return rc;
            if (sz[i])
                CK(cudaMemcpyAsync(ctx->svc_in[i].p, src[i], sz[i], cudaMemcpyHostToDevice, s));
            dev[i] = ctx->svc_in[i].p;
        }
    }
    /* 58 fixed + 3 commas + '}}}' + "srvce":"" + "proto":"" + "port": + 10 digits + "ttl": + '-' and 10 digits */
    const uint64_t cap = n * (uint64_t)(58 + 3 + 3 + 10 + 10 + 7 + 10 + 6 + 11) + srvce_len + proto_len + 16;
    const uint64_t ntiles = (n + TILE - 1) / TILE;
    const size_t totals_off = 128, super_off = (totals_off + ntiles * 4 + 15) & ~(size_t)15;
    const size_t work_bytes = super_off + (ntiles / SUPER + 1) * 8 + 64;
    if ((rc = ensure_dev(ctx, ctx->json_bytes, cap)) || (rc = ensure_dev(ctx, ctx->json_off, (n + 1) * 8)) ||
        (rc = ensure_dev(ctx, ctx->svc_work, work_bytes)))
        return rc;
    uint8_t *wk = (uint8_t *)ctx->svc_work.p;
    CK(cudaMemsetAsync(wk, 0, work_bytes, s));
    if (n == 0)
        CK(cudaMemsetAsync(ctx->json_off.p, 0, 8, s));
    regk_ctx::Slot &slot = ctx->slots[0];
    uint32_t launches = 0;
    if (n) {
        ServiceParams p{};
        p.n = n;
        p.srvce_bytes = (const uint8_t *)dev[0];
        p.srvce_off = (const uint32_t *)dev[1];
        p.proto_bytes = (const uint8_t *)dev[2];
        p.proto_off = (const uint32_t *)dev[3];
        p.port = (const uint32_t *)dev[4];
        p.ttl = (const int32_t *)dev[5];
        p.key_order = (const uint8_t *)dev[6];
        p.out_bytes = (uint8_t *)ctx->json_bytes.p;
        p.out_off = (unsigned long long *)ctx->json_off.p;
        p.out_capacity = cap;
        p.tile_total = (uint32_t *)(wk + totals_off);
        p.super_total = (unsigned long long *)(wk + super_off);
        p.status = (DevStatus *)wk;
        p.srvce_limit = srvce_len;
        p.proto_limit = proto_len;
        const uint64_t mean = 58 + 3 + 3 + 20 + 13 + 17 + (srvce_len + proto_len) / n + 2;
        p.out_cap = (uint32_t)align16(std::min<uint64_t>(mean * TILE * 9 / 8 + 512, 98304));
        const size_t smem = (size_t)p.out_cap + 32;
        if (smem_attr_needs_raise(ctx->device, 3, smem))
            CK(cudaFuncSetAttribute(regk_service_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        CK(cudaEventRecord(slot.ev[0], s));
        regk_service_len_kernel<<<(unsigned)std::min<uint64_t>(ntiles, (uint64_t)ctx->sm_count * 8), TILE, 0, s>>>(p, (uint32_t)ntiles);
        CK(cudaGetLastError());
        regk_service_kernel<<<(unsigned)ntiles, TILE, smem, s>>>(p);
        CK(cudaGetLastError());
        CK(cudaEventRecord(slot.ev[1], s));
        launches = 2;
    }
    CK(cudaMemcpyAsync(slot.h_status, wk, sizeof(DevStatus), cudaMemcpyDeviceToHost, s));
    cudaError_t e = cudaStreamSynchronize(s);
    if (e != cudaSuccess)
        return fail(ctx, REGK_ERR_CUDA, "regk_service_records: kernel execution failed: %s", cudaGetErrorString(e));
    const DevStatus st = *slot.h_status;
    res->n = n;
    res->launches = launches;
    res->bad_bits = st.bad_bits;
    res->first_bad = st.bad_bits ? ~st.first_bad : 0;
    if (n) {
        float ms = 0;
        cudaEventElapsedTime(&ms, slot.ev[0], slot.ev[1]);
        res->kernel_ms = res->json_kernel_ms = ms;
    }
    if (st.overflow)
        return fail(ctx, REGK_ERR_CUDA, "internal error: output capacity bound exceeded");
    if (st.bad_bits)
        return fail(ctx, REGK_ERR_OUT_OF_DOMAIN,
            "service record %llu is outside the supported input domain (REGK_BAD bits 0x%x); no output produced",
            (unsigned long long)res->first_bad, st.bad_bits);
    res->json_total = st.json_total;
    ctx->last_gen++;
    ctx->last_path_off = nullptr;                   /* the payload buffers were reused */
    ctx->last_json_off = nullptr;
    if (out_dev) {
        res->flags = REGK_OUT_DEVICE;
        res->json_bytes = (uint8_t *)ctx->json_bytes.p;
        res->json_off = (uint64_t *)ctx->json_off.p;
        return REGK_OK;
    }
    if ((rc = ensure_host(ctx, ctx->h_json_bytes, st.json_total + 16)) || (rc = ensure_host(ctx, ctx->h_json_off, (n + 1) * 8)))
        return rc;
    if (st.json_total)
        CK(cudaMemcpyAsync(ctx->h_json_bytes.p, ctx->json_bytes.p, st.json_total, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(ctx->h_json_off.p, ctx->json_off.p, (n + 1) * 8, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    res->json_bytes = (uint8_t *)ctx->h_json_bytes.p;
    res->json_off = (uint64_t *)ctx->h_json_off.p;
    return REGK_OK;
}

int regk_jute_frames(regk_ctx *ctx, uint32_t flags, int32_t xid_base, uint32_t zk_flags, regk_frames *out)
{
    regk_jute_opts o{};
    o.op = REGK_ZK_CREATE;
    o.flags = flags;
    o.xid_base = xid_base;
    o.zk_flags = zk_flags;
    return regk_jute_requests(ctx, &o, out);
}

int regk_jute_requests(regk_ctx *ctx, const regk_jute_opts *o, regk_frames *out)
{
    if (!ctx || !o || !out)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_jute_requests: NULL argument");
    memset(out, 0, sizeof *out);
    const bool getdata = o->op == REGK_ZK_GETDATA;
    if (o->op != REGK_ZK_CREATE && o->op != REGK_ZK_DELETE && o->op != REGK_ZK_SETDATA && !getdata)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_jute_requests: op %u is not create (1), delete (2), getData (4) or setData (5)",
            o->op);
    if (o->group > 65536)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_jute_requests: at most 65536 operations per multi transaction");
    if (getdata && o->group != 0)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_jute_requests: getData requests cannot go in a multi transaction (group %u)",
            o->group);
    const bool has_data = o->op != REGK_ZK_DELETE && !getdata;
    if (ctx->pending)
        return fail(ctx, REGK_ERR_STATE, "regk_jute_requests: batches are still in flight; finish them first");
    if (!ctx->last_path_off || (has_data && (!ctx->last_json_off || ctx->last_n != ctx->last_json_n)))
        return fail(ctx, REGK_ERR_STATE, "regk_jute_requests: no finished batch with %s on this context",
            has_data ? "both a path and a payload stream" : "a path stream");
    const FrameSrc src{ctx->last_n, ctx->last_path_bytes, ctx->last_path_off, has_data ? ctx->last_json_bytes : nullptr,
                       has_data ? ctx->last_json_off : nullptr};
    const int rc = frame_requests(ctx, src, o, ctx->jute_bytes, ctx->jute_off, ctx->h_jute_bytes, ctx->h_jute_off, out);
    if (rc == REGK_OK && getdata) {
        ctx->gd_valid = true;
        ctx->gd_gen = ctx->last_gen;
        ctx->gd_xid = o->xid_base;
        ctx->gd_n = ctx->last_n;
    }
    return rc;
}

int regk_decode(regk_ctx *ctx, const regk_decode_in *in, regk_decode_out *out)
{
    if (!ctx || !in || !out)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_decode: NULL argument");
    static_assert(sizeof(regk_decoded) == sizeof(Decoded), "regk_decoded layout");
    memset(out, 0, sizeof *out);
    if (ctx->pending)
        return fail(ctx, REGK_ERR_STATE, "regk_decode: batches are still in flight; finish them first");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    const bool last = in->flags & REGK_DECODE_LAST, in_dev = last || (in->flags & REGK_IN_DEVICE);
    const bool dev_out = in->flags & REGK_OUT_DEVICE;
    uint64_t n = in->n, path_total = in->path_total, json_total = in->json_total;
    const uint8_t *pb = in->path_bytes, *jb = in->json_bytes;
    const uint64_t *po = in->path_off, *jo = in->json_off;
    int rc;
    if (last) {
        if (!ctx->last_path_off && !ctx->last_json_off)
            return fail(ctx, REGK_ERR_STATE, "regk_decode: no finished batch on this context");
        n = ctx->last_path_off ? ctx->last_n : ctx->last_json_n;
        pb = ctx->last_path_off ? ctx->last_path_bytes : nullptr;
        po = (const uint64_t *)ctx->last_path_off;
        jb = ctx->last_json_off ? ctx->last_json_bytes : nullptr;
        jo = (const uint64_t *)ctx->last_json_off;
        unsigned long long tot[2] = {0, 0};
        if (po)
            CK(cudaMemcpyAsync(&tot[0], po + n, 8, cudaMemcpyDeviceToHost, s));
        if (jo)
            CK(cudaMemcpyAsync(&tot[1], jo + n, 8, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        path_total = tot[0];
        json_total = tot[1];
    } else {
        if (n >= (1ull << 32))
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_decode: n must be < 2^32 per call");
        if (n && !po && !jo)
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_decode: neither a path nor a payload stream given");
        if ((po && !pb && n) || (jo && !jb && n))
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_decode: offsets without bytes");
        if (!in_dev) {
            path_total = (po && n) ? po[n] : 0;
            json_total = (jo && n) ? jo[n] : 0;
            /* offsets are used as memory ranges by the kernel: they must be monotone and end at the total */
            for (uint64_t i = 0; i < n; i++)
                if ((po && (po[i] > po[i + 1])) || (jo && (jo[i] > jo[i + 1])))
                    return fail(ctx, REGK_ERR_INVALID_ARG, "regk_decode: offsets are not monotone at record %llu", (unsigned long long)i);
            const void *src[4] = {pb, po, jb, jo};
            const size_t sz[4] = {(size_t)path_total, po ? (size_t)(n + 1) * 8 : 0, (size_t)json_total, jo ? (size_t)(n + 1) * 8 : 0};
            const void *dev[4] = {nullptr, nullptr, nullptr, nullptr};
            for (int i = 0; i < 4; i++) {
                if (!src[i] || !n || ((i == 0 || i == 2) && !src[i + 1]))
                    continue;
                if ((rc = ensure_dev(ctx, ctx->dec_in[i], sz[i] + 16)))
                    return rc;
                if (sz[i])
                    CK(cudaMemcpyAsync(ctx->dec_in[i].p, src[i], sz[i], cudaMemcpyHostToDevice, s));
                dev[i] = ctx->dec_in[i].p;
            }
            pb = (const uint8_t *)dev[0];
            po = (const uint64_t *)dev[1];
            jb = (const uint8_t *)dev[2];
            jo = (const uint64_t *)dev[3];
        }
    }
    if (!po)
        pb = nullptr;
    if (!jo)
        jb = nullptr;
    const uint64_t ports_len = json_total / 2 + 1;
    if ((rc = ensure_dev(ctx, ctx->dec_rec, (n + 1) * sizeof(Decoded))) || (rc = ensure_dev(ctx, ctx->dec_dom, path_total + 16)) ||
        (rc = ensure_dev(ctx, ctx->dec_ports, ports_len * 4 + 16)))
        return rc;
    out->n = n;
    out->flags = dev_out ? REGK_OUT_DEVICE : 0;
    out->dom_bytes_len = path_total;
    out->ports_len = ports_len;
    cudaEvent_t e0 = ctx->slots[0].ev[0], e1 = ctx->slots[0].ev[1];
    if (n) {
        DecodeParams p{};
        p.n = n;
        p.path_bytes = po ? (pb ? pb : (const uint8_t *)ctx->dec_dom.p) : nullptr;     /* an empty stream still has offsets */
        p.path_off = (const unsigned long long *)po;
        p.json_bytes = jo ? (jb ? jb : (const uint8_t *)ctx->dec_dom.p) : nullptr;
        p.json_off = (const unsigned long long *)jo;
        p.host_nodes = in->host_nodes;
        p.out = (Decoded *)ctx->dec_rec.p;
        p.dom_bytes = (uint8_t *)ctx->dec_dom.p;
        p.ports = (uint32_t *)ctx->dec_ports.p;
        /* staging budgets: 9/8 of a tile's mean share of each stream plus slack; streams handed in by the caller
           carry no slack behind their last byte, the library's own buffers have >= 16 bytes */
        p.path_cap = (uint32_t)align16(std::min<uint64_t>(path_total * DEC_TILE / n * 9 / 8 + 1024, 49152));
        p.json_cap = (uint32_t)align16(std::min<uint64_t>(json_total * DEC_TILE / n * 9 / 8 + 1024, 65536));
        const uint64_t slack = (in_dev && !last) ? 0 : 16;     /* a caller's own device buffers end where they end */
        p.path_limit = path_total + slack;
        p.json_limit = json_total + slack;
        /* [path slice, later the result records][slash bitmap][payload slice, later the domain image] (regk_decode.cuh) */
        const size_t dsmem = std::max<size_t>((size_t)p.path_cap + 32, DEC_TILE * sizeof(Decoded)) + ((p.path_cap / 8 + 47) & ~15u) +
            std::max<size_t>(p.json_cap, p.path_cap) + 32 + 16;
        {
            static std::mutex mu;
            static size_t high[64];
            std::lock_guard<std::mutex> lock(mu);
            if (dsmem > high[ctx->device & 63]) {
                CK(cudaFuncSetAttribute(regk_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dsmem));
                high[ctx->device & 63] = dsmem;
            }
        }
        CK(cudaEventRecord(e0, s));
        regk_decode_kernel<<<(unsigned)((n + DEC_TILE - 1) / DEC_TILE), DEC_TILE, dsmem, s>>>(p);
        CK(cudaGetLastError());
        CK(cudaEventRecord(e1, s));
        out->launches = 1;
    }
    cudaError_t e = cudaStreamSynchronize(s);
    if (e != cudaSuccess)
        return fail(ctx, REGK_ERR_CUDA, "regk_decode: kernel execution failed: %s", cudaGetErrorString(e));
    if (n)
        cudaEventElapsedTime(&out->kernel_ms, e0, e1);
    if (dev_out) {
        out->rec = (const regk_decoded *)ctx->dec_rec.p;
        out->dom_bytes = (const uint8_t *)ctx->dec_dom.p;
        out->ports = (const uint32_t *)ctx->dec_ports.p;
        return REGK_OK;
    }
    if ((rc = ensure_host(ctx, ctx->h_dec_rec, (n + 1) * sizeof(Decoded))) || (rc = ensure_host(ctx, ctx->h_dec_dom, path_total + 16)) ||
        (rc = ensure_host(ctx, ctx->h_dec_ports, ports_len * 4 + 16)))
        return rc;
    if (n) {
        CK(cudaMemcpyAsync(ctx->h_dec_rec.p, ctx->dec_rec.p, n * sizeof(Decoded), cudaMemcpyDeviceToHost, s));
        if (po && path_total)
            CK(cudaMemcpyAsync(ctx->h_dec_dom.p, ctx->dec_dom.p, path_total, cudaMemcpyDeviceToHost, s));
        if (jo)
            CK(cudaMemcpyAsync(ctx->h_dec_ports.p, ctx->dec_ports.p, ports_len * 4, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
    }
    out->rec = (const regk_decoded *)ctx->h_dec_rec.p;
    out->dom_bytes = (const uint8_t *)ctx->h_dec_dom.p;
    out->ports = (const uint32_t *)ctx->h_dec_ports.p;
    return REGK_OK;
}

int regk_parent_dirs(regk_ctx *ctx, uint32_t flags, regk_parents *out)
{
    if (!ctx || !out)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_parent_dirs: NULL argument");
    memset(out, 0, sizeof *out);
    if (ctx->pending)
        return fail(ctx, REGK_ERR_STATE, "regk_parent_dirs: batches are still in flight; finish them first");
    if (!ctx->last_path_off || !ctx->last_path_bytes)
        return fail(ctx, REGK_ERR_STATE, "regk_parent_dirs: no finished batch with a path stream on this context");
    const uint64_t n = ctx->last_n;
    if (n >= 0xFFFFFFFEull)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_parent_dirs: batch too large");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    const bool dev_out = flags & REGK_OUT_DEVICE;
    out->n = n;
    out->flags = dev_out ? REGK_OUT_DEVICE : 0;
    if (n == 0)
        return REGK_OK;
    int rc;
    if ((rc = ensure_host(ctx, ctx->h_par_count, 8)))
        return rc;
    if (!ctx->par_ev[0]) {
        CK(cudaEventCreate(&ctx->par_ev[0]));
        CK(cudaEventCreate(&ctx->par_ev[1]));
    }
    cudaEvent_t e0 = ctx->par_ev[0], e1 = ctx->par_ev[1];
    ParentParams p{};
    if ((rc = enqueue_parent_pass(ctx, ctx->par_len, ctx->par_slot, ctx->par_table, ctx->par_totals, ctx->par_unique, n, e0, &p)))
        return rc;
    CK(cudaEventRecord(e1, s));
    CK(cudaMemcpyAsync(ctx->h_par_count.p, p.n_unique, 8, cudaMemcpyDeviceToHost, s));
    cudaError_t e = cudaStreamSynchronize(s);
    float ms = 0;
    if (e == cudaSuccess)
        cudaEventElapsedTime(&ms, e0, e1);
    if (e != cudaSuccess)
        return fail(ctx, REGK_ERR_CUDA, "regk_parent_dirs: kernel execution failed: %s", cudaGetErrorString(e));
    const uint64_t nu = *(const unsigned long long *)ctx->h_par_count.p;
    out->n_unique = nu;
    out->launches = 3;
    out->kernel_ms = ms;
    if (dev_out) {
        out->parent_len = p.parent_len;
        out->unique_first = (const uint64_t *)p.unique_first;
        return REGK_OK;
    }
    if ((rc = ensure_host(ctx, ctx->h_par_len, n * 4)) || (rc = ensure_host(ctx, ctx->h_par_unique, nu * 8 + 8)))
        return rc;
    CK(cudaMemcpyAsync(ctx->h_par_len.p, p.parent_len, n * 4, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(ctx->h_par_unique.p, p.unique_first, nu * 8, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    out->parent_len = (const uint32_t *)ctx->h_par_len.p;
    out->unique_first = (const uint64_t *)ctx->h_par_unique.p;
    return REGK_OK;
}

int regk_mkdirp_dirs(regk_ctx *ctx, uint32_t flags, regk_dirs *out)
{
    if (!ctx || !out)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_mkdirp_dirs: NULL argument");
    memset(out, 0, sizeof *out);
    if (ctx->pending)
        return fail(ctx, REGK_ERR_STATE, "regk_mkdirp_dirs: batches are still in flight; finish them first");
    if (!ctx->last_path_off || !ctx->last_path_bytes)
        return fail(ctx, REGK_ERR_STATE, "regk_mkdirp_dirs: no finished batch with a path stream on this context");
    const uint64_t n = ctx->last_n;
    if (n >= 0xFFFFFFFEull)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_mkdirp_dirs: batch too large");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    const bool dev_out = flags & REGK_OUT_DEVICE;
    ctx->mk_valid = false;
    DevBuf *mk = ctx->mk;
    int rc;
    if ((rc = ensure_host(ctx, ctx->h_mk_count, 64)) || (rc = ensure_dev(ctx, mk[regk_ctx::MK_COUNT], 64)))
        return rc;
    for (auto &ev : ctx->mk_ev)
        if (!ev)
            CK(cudaEventCreate(&ev));
    unsigned long long *hc = (unsigned long long *)ctx->h_mk_count.p;
    unsigned long long *dc = (unsigned long long *)mk[regk_ctx::MK_COUNT].p;
    auto read_counters = [&](const void *src, size_t bytes) -> int {
        CK(cudaMemcpyAsync(hc, src, bytes, cudaMemcpyDeviceToHost, s));
        const cudaError_t e = cudaStreamSynchronize(s);
        if (e != cudaSuccess)
            return fail(ctx, REGK_ERR_CUDA, "regk_mkdirp_dirs: kernel execution failed: %s", cudaGetErrorString(e));
        return REGK_OK;
    };
    std::vector<uint64_t> depth_off(1, 0);
    uint64_t n_invalid = 0, n_dirs = 0, bytes = 0;
    uint32_t launches = 0;
    float ms[3] = {0, 0, 0};
    if (n) {
        /* 1. the distinct immediate directories, on buffers of its own (regk_parent_dirs' results stay as they are) */
        ParentParams pp{};
        if ((rc = enqueue_parent_pass(ctx, mk[regk_ctx::MK_PLEN], mk[regk_ctx::MK_PSLOT], mk[regk_ctx::MK_PTABLE],
                 mk[regk_ctx::MK_PTOTALS], mk[regk_ctx::MK_PUNIQUE], n, ctx->mk_ev[0], &pp)))
            return rc;
        launches += 3;
        CK(cudaEventRecord(ctx->mk_ev[1], s));
        if ((rc = read_counters(pp.n_unique, 8)))
            return rc;
        const uint64_t nu = hc[0];
        /* workspace for up to nu items per pass: flags, two work lists, two-level totals of two counts */
        const uint64_t ntiles = (nu + MK_TILE - 1) / MK_TILE, tt = align16(ntiles * 4), st = (ntiles / SUPER + 1) * 8;
        const size_t totals_bytes = 2 * tt + 2 * st + 16;
        if ((rc = ensure_dev(ctx, mk[regk_ctx::MK_FLAGS], nu + 16)) || (rc = ensure_dev(ctx, mk[regk_ctx::MK_LIST0], nu * 16 + 16)) ||
            (rc = ensure_dev(ctx, mk[regk_ctx::MK_LIST1], nu * 16 + 16)) || (rc = ensure_dev(ctx, mk[regk_ctx::MK_TOTALS], totals_bytes)) ||
            (rc = ensure_dev(ctx, mk[regk_ctx::MK_INVALID], nu * 8 + 8)))
            return rc;
        uint8_t *tb = (uint8_t *)mk[regk_ctx::MK_TOTALS].p;
        MkdirpParams p{};
        p.path_bytes = ctx->last_path_bytes;
        p.path_off = ctx->last_path_off;
        p.parent_len = pp.parent_len;
        p.unique_first = pp.unique_first;
        p.n_unique = nu;
        p.flags = (uint8_t *)mk[regk_ctx::MK_FLAGS].p;
        p.tile_a = (uint32_t *)tb;
        p.tile_b = (uint32_t *)(tb + tt);
        p.super_a = (unsigned long long *)(tb + 2 * tt);
        p.super_b = (unsigned long long *)(tb + 2 * tt + st);
        p.counters = dc;
        p.invalid = (unsigned long long *)mk[regk_ctx::MK_INVALID].p;
        uint4 *list[2] = {(uint4 *)mk[regk_ctx::MK_LIST0].p, (uint4 *)mk[regk_ctx::MK_LIST1].p};
        CK(cudaMemsetAsync(dc, 0, 64, s));
        /* 2. root / invalid / depth of each; the invalid list and the depth-1 work list */
        p.m = nu;
        p.list_out = list[0];
        CK(cudaMemsetAsync(tb, 0, totals_bytes, s));
        regk_mkdirp_classify_kernel<<<(unsigned)ntiles, MK_TILE, 0, s>>>(p);
        regk_mkdirp_split_kernel<false><<<(unsigned)ntiles, MK_TILE, 0, s>>>(p);
        CK(cudaGetLastError());
        launches += 2;
        if ((rc = read_counters(dc, 32)))
            return rc;
        n_invalid = hc[0];
        uint64_t m = hc[1];
        const uint64_t entries = hc[3];
        /* 3. the table: 64-bit slots, at most 2/3 full even before duplicates merge; "mkdirp_tight_table" = 1 sizes it
           to the smallest power of two above the entry count (long probe chains; testing) */
        uint64_t slots = 1024;
        if (opt_get(ctx, "mkdirp_tight_table", 0)) {
            slots = 2;
            while (slots <= entries)
                slots <<= 1;
        } else {
            while (slots < entries + entries / 2)
                slots <<= 1;
        }
        if (slots > (1ull << 32))
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_mkdirp_dirs: %llu directory entries are too many for one table",
                (unsigned long long)entries);
        if ((rc = ensure_dev(ctx, mk[regk_ctx::MK_TABLE], slots * 8)) || (rc = ensure_dev(ctx, mk[regk_ctx::MK_DREC], entries * 8 + 8)) ||
            (rc = ensure_dev(ctx, mk[regk_ctx::MK_DLEN], entries * 4 + 8)))
            return rc;
        p.table = (unsigned long long *)mk[regk_ctx::MK_TABLE].p;
        p.mask = (uint32_t)(slots - 1);
        p.dir_rec = (unsigned long long *)mk[regk_ctx::MK_DREC].p;
        p.dir_len = (uint32_t *)mk[regk_ctx::MK_DLEN].p;
        CK(cudaMemsetAsync(p.table, 0, slots * 8, s));
        /* 4. one depth at a time: extend + insert, mark, split; the host reads how many directories and entries remain */
        for (int cur = 0; m; cur ^= 1) {
            const uint64_t mt = (m + MK_TILE - 1) / MK_TILE;
            p.m = m;
            p.list_in = list[cur];
            p.list_out = list[cur ^ 1];
            p.dir_base = n_dirs;
            CK(cudaMemsetAsync(tb, 0, totals_bytes, s));
            regk_mkdirp_insert_kernel<<<(unsigned)((m + 255) / 256), 256, 0, s>>>(p);
            regk_mkdirp_mark_kernel<<<(unsigned)mt, MK_TILE, 0, s>>>(p);
            regk_mkdirp_split_kernel<true><<<(unsigned)mt, MK_TILE, 0, s>>>(p);
            CK(cudaGetLastError());
            launches += 3;
            if ((rc = read_counters(dc, 24)))
                return rc;
            n_dirs += hc[0];
            depth_off.push_back(n_dirs);
            m = hc[1];
            bytes = hc[2];
        }
        CK(cudaEventRecord(ctx->mk_ev[2], s));
        /* 5. dir_off and the packed bytes */
        const uint64_t dt = (n_dirs + MK_TILE - 1) / MK_TILE, dtt = dt * 8, dst = (dt / SUPER + 1) * 8;
        if ((rc = ensure_dev(ctx, mk[regk_ctx::MK_DBYTES], bytes + 16)) || (rc = ensure_dev(ctx, mk[regk_ctx::MK_DOFF], (n_dirs + 1) * 8)) ||
            (rc = ensure_dev(ctx, mk[regk_ctx::MK_TOTALS], dtt + dst + 16)))
            return rc;
        if (n_dirs) {
            MkGatherParams g{};
            g.n_dirs = n_dirs;
            g.path_bytes = ctx->last_path_bytes;
            g.path_off = ctx->last_path_off;
            g.dir_rec = p.dir_rec;
            g.dir_len = p.dir_len;
            g.tile_total = (unsigned long long *)mk[regk_ctx::MK_TOTALS].p;
            g.super_total = (unsigned long long *)((uint8_t *)mk[regk_ctx::MK_TOTALS].p + dtt);
            g.dir_bytes = (uint8_t *)mk[regk_ctx::MK_DBYTES].p;
            g.dir_off = (unsigned long long *)mk[regk_ctx::MK_DOFF].p;
            CK(cudaMemsetAsync(g.super_total, 0, dst, s));
            regk_mkdirp_len_kernel<<<(unsigned)dt, MK_TILE, 0, s>>>(g);
            regk_mkdirp_gather_kernel<<<(unsigned)dt, MK_TILE, 0, s>>>(g);
            CK(cudaGetLastError());
            launches += 2;
        } else {
            CK(cudaMemsetAsync(mk[regk_ctx::MK_DOFF].p, 0, 8, s));
        }
        CK(cudaEventRecord(ctx->mk_ev[3], s));
        const cudaError_t e = cudaStreamSynchronize(s);
        if (e != cudaSuccess)
            return fail(ctx, REGK_ERR_CUDA, "regk_mkdirp_dirs: kernel execution failed: %s", cudaGetErrorString(e));
        for (int k = 0; k < 3; k++)
            cudaEventElapsedTime(&ms[k], ctx->mk_ev[k], ctx->mk_ev[k + 1]);
    } else {
        if ((rc = ensure_dev(ctx, mk[regk_ctx::MK_DOFF], 8)) || (rc = ensure_dev(ctx, mk[regk_ctx::MK_DBYTES], 16)) ||
            (rc = ensure_dev(ctx, mk[regk_ctx::MK_DREC], 8)) || (rc = ensure_dev(ctx, mk[regk_ctx::MK_DLEN], 8)) ||
            (rc = ensure_dev(ctx, mk[regk_ctx::MK_INVALID], 8)))
            return rc;
        CK(cudaMemsetAsync(mk[regk_ctx::MK_DOFF].p, 0, 8, s));
    }
    /* depth_off was counted on the host; the device result gets a copy */
    const size_t nd1 = depth_off.size();
    if ((rc = ensure_host(ctx, ctx->h_mk_depth, nd1 * 8)) || (rc = ensure_dev(ctx, mk[regk_ctx::MK_DEPTH], nd1 * 8)))
        return rc;
    memcpy(ctx->h_mk_depth.p, depth_off.data(), nd1 * 8);
    CK(cudaMemcpyAsync(mk[regk_ctx::MK_DEPTH].p, ctx->h_mk_depth.p, nd1 * 8, cudaMemcpyHostToDevice, s));
    CK(cudaStreamSynchronize(s));
    ctx->mk_valid = true;
    ctx->mk_n_dirs = n_dirs;
    ctx->mk_bytes = bytes;
    out->n = n;
    out->n_dirs = n_dirs;
    out->n_invalid = n_invalid;
    out->flags = dev_out ? REGK_OUT_DEVICE : 0;
    out->launches = launches;
    out->max_depth = (uint32_t)(nd1 - 1);
    out->dir_bytes_len = bytes;
    out->parent_ms = ms[0];
    out->closure_ms = ms[1];
    out->gather_ms = ms[2];
    out->kernel_ms = ms[0] + ms[1] + ms[2];
    const void *dsrc[6] = {mk[regk_ctx::MK_DREC].p, mk[regk_ctx::MK_DLEN].p, mk[regk_ctx::MK_DEPTH].p, mk[regk_ctx::MK_DBYTES].p,
                           mk[regk_ctx::MK_DOFF].p, mk[regk_ctx::MK_INVALID].p};
    if (!dev_out) {
        HostBuf *hb[6] = {&ctx->h_mk_drec, &ctx->h_mk_dlen, &ctx->h_mk_depth, &ctx->h_mk_dbytes, &ctx->h_mk_doff, &ctx->h_mk_invalid};
        const size_t sz[6] = {n_dirs * 8, n_dirs * 4, 0, bytes, (n_dirs + 1) * 8, n_invalid * 8};
        for (int k = 0; k < 6; k++) {
            if (k == 2)
                continue;                               /* already on the host */
            if ((rc = ensure_host(ctx, *hb[k], sz[k] + 16)))
                return rc;
            if (sz[k])
                CK(cudaMemcpyAsync(hb[k]->p, dsrc[k], sz[k], cudaMemcpyDeviceToHost, s));
            dsrc[k] = hb[k]->p;
        }
        dsrc[2] = ctx->h_mk_depth.p;
        CK(cudaStreamSynchronize(s));
    }
    out->dir_rec = (const uint64_t *)dsrc[0];
    out->dir_len = (const uint32_t *)dsrc[1];
    out->depth_off = (const uint64_t *)dsrc[2];
    out->dir_bytes = (const uint8_t *)dsrc[3];
    out->dir_off = (const uint64_t *)dsrc[4];
    out->invalid = (const uint64_t *)dsrc[5];
    return REGK_OK;
}

int regk_mkdirp_requests(regk_ctx *ctx, int32_t xid_base, uint32_t zk_flags, uint32_t flags, regk_frames *out)
{
    if (!ctx || !out)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_mkdirp_requests: NULL argument");
    memset(out, 0, sizeof *out);
    if (ctx->pending)
        return fail(ctx, REGK_ERR_STATE, "regk_mkdirp_requests: batches are still in flight; finish them first");
    if (!ctx->mk_valid)
        return fail(ctx, REGK_ERR_STATE, "regk_mkdirp_requests: no directory set on this context; call regk_mkdirp_dirs first");
    CK(cudaSetDevice(ctx->device));
    const uint64_t nd = ctx->mk_n_dirs;
    int rc;
    /* CreateRequest with an empty data buffer: the payload offsets are all zero */
    if ((rc = ensure_dev(ctx, ctx->mk[regk_ctx::MK_ZERO], (nd + 1) * 8)))
        return rc;
    CK(cudaMemsetAsync(ctx->mk[regk_ctx::MK_ZERO].p, 0, (nd + 1) * 8, ctx->stream));
    regk_jute_opts o{};
    o.op = REGK_ZK_CREATE;
    o.flags = flags;
    o.xid_base = xid_base;
    o.zk_flags = zk_flags;
    FrameSrc src{nd, (const uint8_t *)ctx->mk[regk_ctx::MK_DBYTES].p, (const unsigned long long *)ctx->mk[regk_ctx::MK_DOFF].p,
                 (const uint8_t *)ctx->mk[regk_ctx::MK_DBYTES].p, (const unsigned long long *)ctx->mk[regk_ctx::MK_ZERO].p};
    src.who = "regk_mkdirp_requests";
    return frame_requests(ctx, src, &o, ctx->mk[regk_ctx::MK_FBYTES], ctx->mk[regk_ctx::MK_FOFF], ctx->h_mk_fbytes, ctx->h_mk_foff, out);
}

/* regk_reconcile (st == NULL) and regk_reconcile_owned: one implementation, the same four passes; `rep` / `n_rep` receive
   the replace list of the owned call */
static int reconcile_run(regk_ctx *ctx, const regk_decode_in *in, const regk_node_stat *st, uint32_t flags, regk_delta *out,
    const uint64_t **rep, uint64_t *n_rep, const char *who)
{
    ctx->rc_valid = false;
    if (in->flags & REGK_DECODE_LAST)
        return fail(ctx, REGK_ERR_INVALID_ARG, "%s: REGK_DECODE_LAST names no snapshot; pass the snapshot's streams", who);
    if (ctx->pending)
        return fail(ctx, REGK_ERR_STATE, "%s: batches are still in flight; finish them first", who);
    if (!ctx->last_path_off || !ctx->last_json_off || ctx->last_n != ctx->last_json_n)
        return fail(ctx, REGK_ERR_STATE, "%s: no finished batch with both a path and a payload stream on this context "
                                         "(an empty batch or a REGK_JOB_STEP result leaves none)", who);
    const uint64_t n = ctx->last_n, m = in->n;
    if (n >= 0xFFFFFFFFull || m >= 0xFFFFFFFFull)
        return fail(ctx, REGK_ERR_INVALID_ARG, "%s: %llu records and %llu nodes: both must be below 2^32 - 1", who,
            (unsigned long long)n, (unsigned long long)m);
    const bool in_dev = in->flags & REGK_IN_DEVICE, dev_out = flags & REGK_OUT_DEVICE;
    const uint8_t *pb = in->path_bytes, *jb = in->json_bytes;
    const uint64_t *po = in->path_off, *jo = in->json_off;
    uint64_t path_total = m ? in->path_total : 0, json_total = m ? in->json_total : 0;
    if (m && (!po || !jo))
        return fail(ctx, REGK_ERR_INVALID_ARG, "%s: a snapshot of %llu nodes needs path and data offsets", who, (unsigned long long)m);
    const int32_t *sver = st ? st->version : nullptr;
    const int64_t *sown = st ? st->ephemeral_owner : nullptr;
    if (st && m && (!sver || !sown))
        return fail(ctx, REGK_ERR_INVALID_ARG, "%s: a snapshot of %llu nodes needs a version and an owner per node", who,
            (unsigned long long)m);
    if (st && m && in_dev && (((uintptr_t)sver & 3u) || ((uintptr_t)sown & 7u)))
        return fail(ctx, REGK_ERR_INVALID_ARG, "%s: misaligned device stats (version needs 4-byte, ephemeral_owner 8-byte alignment)", who);
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    DevBuf *rb = ctx->rc;
    int rc;
    if (m && !in_dev) {
        path_total = po[m];
        json_total = jo[m];
        /* offsets become memory ranges in the kernels: monotone, each node below 4 GiB, ending at the totals */
        for (uint64_t j = 0; j < m; j++)
            if (po[j] > po[j + 1] || jo[j] > jo[j + 1] || po[j + 1] - po[j] > 0xFFFFFFFFull || jo[j + 1] - jo[j] > 0xFFFFFFFFull)
                return fail(ctx, REGK_ERR_INVALID_ARG, "%s: snapshot offsets are not monotone at node %llu", who,
                    (unsigned long long)j);
        if ((path_total && !pb) || (json_total && !jb))
            return fail(ctx, REGK_ERR_INVALID_ARG, "%s: snapshot offsets without bytes", who);
        const void *src[6] = {pb, po, jb, jo, sver, sown};
        const size_t sz[6] = {(size_t)path_total, (size_t)(m + 1) * 8, (size_t)json_total, (size_t)(m + 1) * 8, (size_t)m * 4, (size_t)m * 8};
        for (int k = 0; k < (st ? 6 : 4); k++) {
            if ((rc = ensure_dev(ctx, rb[regk_ctx::RC_IN_PB + k], sz[k] + 16)))
                return rc;
            if (sz[k])
                CK(cudaMemcpyAsync(rb[regk_ctx::RC_IN_PB + k].p, src[k], sz[k], cudaMemcpyHostToDevice, s));
        }
        pb = (const uint8_t *)rb[regk_ctx::RC_IN_PB].p;
        po = (const uint64_t *)rb[regk_ctx::RC_IN_PO].p;
        jb = (const uint8_t *)rb[regk_ctx::RC_IN_JB].p;
        jo = (const uint64_t *)rb[regk_ctx::RC_IN_JO].p;
        if (st) {
            sver = (const int32_t *)rb[regk_ctx::RC_IN_VER].p;
            sown = (const int64_t *)rb[regk_ctx::RC_IN_OWN].p;
        }
    } else if (m) {
        if ((path_total && !pb) || (json_total && !jb))
            return fail(ctx, REGK_ERR_INVALID_ARG, "%s: snapshot offsets without bytes", who);
        if (((uintptr_t)pb & 3u) || ((uintptr_t)jb & 3u) || ((uintptr_t)po & 7u) || ((uintptr_t)jo & 7u))
            return fail(ctx, REGK_ERR_INVALID_ARG, "%s: misaligned device snapshot (bytes need 4-byte, offsets 8-byte alignment)", who);
    }
    /* an empty stream is never read; its kernels still get a valid pointer */
    if ((rc = ensure_dev(ctx, rb[regk_ctx::RC_IN_PB], 16)) || (rc = ensure_dev(ctx, rb[regk_ctx::RC_IN_JB], 16)))
        return rc;
    if (!pb)
        pb = (const uint8_t *)rb[regk_ctx::RC_IN_PB].p;
    if (!jb)
        jb = (const uint8_t *)rb[regk_ctx::RC_IN_JB].p;
    /* the batch's totals */
    unsigned long long tot[2] = {0, 0};
    CK(cudaMemcpyAsync(&tot[0], ctx->last_path_off + n, 8, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(&tot[1], ctx->last_json_off + n, 8, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    /* tables: at most half full; "reconcile_tight_table" = 1: the smallest power of two above the entries */
    const bool tight = opt_get(ctx, "reconcile_tight_table", 0) != 0;
    auto table_slots = [tight](uint64_t entries) {
        uint64_t slots = tight ? 2 : 1024;
        while (tight ? slots <= entries : slots < 2 * entries)
            slots <<= 1;
        return slots;
    };
    const uint64_t so = table_slots(m), sd = table_slots(n);
    const uint64_t tiles_r = (n + RC_TILE - 1) / RC_TILE, tiles_o = (m + RC_TILE - 1) / RC_TILE;
    const size_t ttr = align16(tiles_r * 4), str = (tiles_r / SUPER + 1) * 8, tto = align16(tiles_o * 4), sto = (tiles_o / SUPER + 1) * 8;
    const size_t totals_bytes = RC_NREC_LISTS * (ttr + str) + tto + sto;
    const size_t counters_bytes = RC_NCOUNTERS * 8;
    if ((rc = ensure_dev(ctx, rb[regk_ctx::RC_TOBS], so * 4)) || (rc = ensure_dev(ctx, rb[regk_ctx::RC_TDES], sd * 4)) ||
        (rc = ensure_dev(ctx, rb[regk_ctx::RC_SLOTO], m * 4 + 16)) || (rc = ensure_dev(ctx, rb[regk_ctx::RC_HASHO], m * 4 + 16)) ||
        (rc = ensure_dev(ctx, rb[regk_ctx::RC_SLOTD], n * 4)) || (rc = ensure_dev(ctx, rb[regk_ctx::RC_CLS], n + 16)) ||
        (rc = ensure_dev(ctx, rb[regk_ctx::RC_MATCH], n * 8)) || (rc = ensure_dev(ctx, rb[regk_ctx::RC_OBSCLS], m + 16)) ||
        (rc = ensure_dev(ctx, rb[regk_ctx::RC_TOTALS], totals_bytes)) || (rc = ensure_dev(ctx, rb[regk_ctx::RC_COUNT], counters_bytes)) ||
        (rc = ensure_host(ctx, ctx->h_rc_count, counters_bytes)))
        return rc;
    for (int l = 0; l < RC_NLISTS; l++)
        if ((rc = ensure_dev(ctx, rb[regk_ctx::RC_LIST0 + l], (l == RC_LDELETE ? m : n) * 8 + 8)))
            return rc;
    for (int k = 0; k < RC_NGATHERS; k++)
        if ((rc = ensure_dev(ctx, rb[regk_ctx::RC_LEN0 + k], (k == RC_GDELETE ? m : n) * 4 + 8)))
            return rc;
    for (int k = 0; st && k < RC_NVER; k++)
        if ((rc = ensure_dev(ctx, rb[regk_ctx::RC_VER0 + k], (k == RC_VDELETE ? m : n) * 4 + 8)))
            return rc;
    for (auto &ev : ctx->rc_ev)
        if (!ev)
            CK(cudaEventCreate(&ev));
    ReconcileParams p{};
    p.n = n;
    p.m = m;
    p.d_path = ctx->last_path_bytes;
    p.d_path_off = ctx->last_path_off;
    p.d_json = ctx->last_json_bytes;
    p.d_json_off = ctx->last_json_off;
    p.d_path_limit = tot[0] + 16;                   /* every stream buffer of this library has >= 16 bytes of slack */
    p.d_json_limit = tot[1] + 16;
    p.o_path = pb;
    p.o_path_off = (const unsigned long long *)po;
    p.o_json = jb;
    p.o_json_off = (const unsigned long long *)jo;
    p.o_path_total = path_total;                    /* a caller's device buffers end where they end */
    p.o_json_total = json_total;
    p.validate = in_dev ? 1u : 0u;
    if (st) {
        p.o_version = sver;
        p.o_owner = (const long long *)sown;
        p.want = st->zk_flags == 1u ? (long long)st->session : 0ll;
        for (int k = 0; k < RC_NVER; k++)
            p.ver[k] = (int32_t *)rb[regk_ctx::RC_VER0 + k].p;
    }
    p.mask_o = (uint32_t)(so - 1);
    p.mask_d = (uint32_t)(sd - 1);
    p.t_obs = (uint32_t *)rb[regk_ctx::RC_TOBS].p;
    p.t_des = (uint32_t *)rb[regk_ctx::RC_TDES].p;
    p.slot_obs = (uint32_t *)rb[regk_ctx::RC_SLOTO].p;
    p.hash_obs = (uint32_t *)rb[regk_ctx::RC_HASHO].p;
    p.slot_des = (uint32_t *)rb[regk_ctx::RC_SLOTD].p;
    p.cls = (uint8_t *)rb[regk_ctx::RC_CLS].p;
    p.match = (unsigned long long *)rb[regk_ctx::RC_MATCH].p;
    p.obs_cls = (uint8_t *)rb[regk_ctx::RC_OBSCLS].p;
    uint8_t *tb = (uint8_t *)rb[regk_ctx::RC_TOTALS].p;
    for (int l = 0; l < RC_NLISTS; l++) {
        const bool del = l == RC_LDELETE;
        p.tile_total[l] = (uint32_t *)(tb + (size_t)l * (ttr + str));
        p.super_total[l] = (unsigned long long *)(tb + (size_t)l * (ttr + str) + (del ? tto : ttr));
        p.list[l] = (unsigned long long *)rb[regk_ctx::RC_LIST0 + l].p;
    }
    for (int k = 0; k < RC_NGATHERS; k++)
        p.len[k] = (uint32_t *)rb[regk_ctx::RC_LEN0 + k].p;
    p.counters = (unsigned long long *)rb[regk_ctx::RC_COUNT].p;
    p.tiles_r = (uint32_t)tiles_r;
    CK(cudaMemsetAsync(p.t_obs, 0, so * 4, s));
    CK(cudaMemsetAsync(p.t_des, 0, sd * 4, s));
    CK(cudaMemsetAsync(tb, 0, totals_bytes, s));
    CK(cudaMemsetAsync(p.counters, 0, counters_bytes, s));
    CK(cudaMemsetAsync(p.counters, 0xFF, 16, s));   /* no bad node, no duplicate node */
    CK(cudaEventRecord(ctx->rc_ev[0], s));
    uint32_t launches = 0;
    if (m) {
        regk_reconcile_insert_kernel<<<(unsigned)((m + 255) / 256), 256, 0, s>>>(p);
        launches++;
    }
    regk_reconcile_desired_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(p);
    regk_reconcile_mark_kernel<<<(unsigned)(tiles_r + tiles_o), RC_TILE, 0, s>>>(p);
    regk_reconcile_compact_kernel<<<(unsigned)(tiles_r + tiles_o), RC_TILE, 0, s>>>(p);
    CK(cudaGetLastError());
    launches += 3;
    unsigned long long *hc = (unsigned long long *)ctx->h_rc_count.p;
    CK(cudaMemcpyAsync(hc, p.counters, counters_bytes, cudaMemcpyDeviceToHost, s));
    cudaError_t e = cudaStreamSynchronize(s);
    if (e != cudaSuccess)
        return fail(ctx, REGK_ERR_CUDA, "%s: kernel execution failed: %s", who, cudaGetErrorString(e));
    if (hc[RC_C_BAD] != ~0ull)
        return fail(ctx, REGK_ERR_INVALID_ARG, "%s: snapshot offsets are not monotone or reach past the totals at node %llu", who,
            hc[RC_C_BAD]);
    if (hc[RC_C_DUPNODE] != ~0ull)
        return fail(ctx, REGK_ERR_INVALID_ARG, "%s: snapshot node %llu has the path of an earlier node; a registry cannot "
                                               "hold two nodes with one path", who, hc[RC_C_DUPNODE]);
    uint64_t cnt[RC_NLISTS];
    for (int l = 0; l < RC_NLISTS; l++)
        cnt[l] = hc[RC_C_COUNT + l];
    if (n == 0)
        cnt[RC_LCREATE] = cnt[RC_LUPDATE] = cnt[RC_LDUP] = cnt[RC_LREPLACE] = 0;
    if (m == 0)
        cnt[RC_LDELETE] = 0;
    /* the request sets, packed: create paths, create payloads, update paths, update payloads, delete paths, replace
       paths, replace payloads */
    const int g_list[RC_NGATHERS] = {RC_LCREATE, RC_LCREATE, RC_LUPDATE, RC_LUPDATE, RC_LDELETE, RC_LREPLACE, RC_LREPLACE};
    const uint8_t *g_src[RC_NGATHERS] = {p.d_path, p.d_json, p.d_path, p.d_json, p.o_path, p.d_path, p.d_json};
    const unsigned long long *g_off[RC_NGATHERS] = {p.d_path_off, p.d_json_off, p.d_path_off, p.d_json_off, p.o_path_off,
                                                    p.d_path_off, p.d_json_off};
    uint64_t gmax = 0;
    for (int g = 0; g < RC_NGATHERS; g++)
        gmax = std::max<uint64_t>(gmax, cnt[g_list[g]]);
    const uint64_t gt = (gmax + MK_TILE - 1) / MK_TILE;
    if ((rc = ensure_dev(ctx, rb[regk_ctx::RC_GTOTALS], gt * 8 + (gt / SUPER + 1) * 8 + 16)))
        return rc;
    for (int g = 0; g < RC_NGATHERS; g++) {
        const uint64_t c = cnt[g_list[g]], bytes = hc[RC_C_BYTES + g];
        DevBuf &gb = rb[regk_ctx::RC_G0B + 2 * g], &go = rb[regk_ctx::RC_G0B + 2 * g + 1];
        if ((rc = ensure_dev(ctx, gb, bytes + 16)) || (rc = ensure_dev(ctx, go, (c + 1) * 8)))
            return rc;
        if (!c) {
            CK(cudaMemsetAsync(go.p, 0, 8, s));
            continue;
        }
        const uint64_t dt = (c + MK_TILE - 1) / MK_TILE;
        MkGatherParams gp{};
        gp.n_dirs = c;
        gp.path_bytes = g_src[g];
        gp.path_off = g_off[g];
        gp.dir_rec = p.list[g_list[g]];
        gp.dir_len = p.len[g];
        gp.tile_total = (unsigned long long *)rb[regk_ctx::RC_GTOTALS].p;
        gp.super_total = gp.tile_total + dt;
        gp.dir_bytes = (uint8_t *)gb.p;
        gp.dir_off = (unsigned long long *)go.p;
        CK(cudaMemsetAsync(gp.super_total, 0, (dt / SUPER + 1) * 8, s));
        regk_mkdirp_len_kernel<<<(unsigned)dt, MK_TILE, 0, s>>>(gp);
        regk_mkdirp_gather_kernel<<<(unsigned)dt, MK_TILE, 0, s>>>(gp);
        CK(cudaGetLastError());
        launches += 2;
    }
    CK(cudaEventRecord(ctx->rc_ev[1], s));
    e = cudaStreamSynchronize(s);
    if (e != cudaSuccess)
        return fail(ctx, REGK_ERR_CUDA, "%s: kernel execution failed: %s", who, cudaGetErrorString(e));
    float ms = 0;
    cudaEventElapsedTime(&ms, ctx->rc_ev[0], ctx->rc_ev[1]);
    const int NOUT = 3 + RC_NLISTS;                 /* cls, match, obs_cls, then the lists */
    const void *dsrc[NOUT] = {p.cls, p.match, p.obs_cls};
    for (int l = 0; l < RC_NLISTS; l++)
        dsrc[3 + l] = p.list[l];
    if (!dev_out) {
        HostBuf *hb[NOUT] = {&ctx->h_rc_cls, &ctx->h_rc_match, &ctx->h_rc_obscls};
        size_t sz[NOUT] = {n, n * 8, m};
        for (int l = 0; l < RC_NLISTS; l++) {
            hb[3 + l] = &ctx->h_rc_list[l];
            sz[3 + l] = cnt[l] * 8;
        }
        for (int k = 0; k < NOUT; k++) {
            if ((rc = ensure_host(ctx, *hb[k], sz[k] + 16)))
                return rc;
            if (sz[k])
                CK(cudaMemcpyAsync(hb[k]->p, dsrc[k], sz[k], cudaMemcpyDeviceToHost, s));
            dsrc[k] = hb[k]->p;
        }
        CK(cudaStreamSynchronize(s));
    }
    ctx->rc_valid = true;
    ctx->rc_owned = st != nullptr;
    ctx->rc_zk_flags = st ? st->zk_flags : 0u;
    for (int l = 0; l < RC_NLISTS; l++)
        ctx->rc_count[l] = cnt[l];
    out->n = n;
    out->m = m;
    out->n_create = cnt[RC_LCREATE];
    out->n_update = cnt[RC_LUPDATE];
    out->n_dup = cnt[RC_LDUP];
    out->n_delete = cnt[RC_LDELETE];
    out->n_same = n - out->n_create - out->n_update - out->n_dup - cnt[RC_LREPLACE];
    out->flags = dev_out ? REGK_OUT_DEVICE : 0;
    out->launches = launches;
    out->cls = (const uint8_t *)dsrc[0];
    out->match = (const uint64_t *)dsrc[1];
    out->obs_cls = (const uint8_t *)dsrc[2];
    out->create = (const uint64_t *)dsrc[3 + RC_LCREATE];
    out->update = (const uint64_t *)dsrc[3 + RC_LUPDATE];
    out->dup = (const uint64_t *)dsrc[3 + RC_LDUP];
    out->del = (const uint64_t *)dsrc[3 + RC_LDELETE];
    out->kernel_ms = ms;
    if (rep) {
        *rep = (const uint64_t *)dsrc[3 + RC_LREPLACE];
        *n_rep = cnt[RC_LREPLACE];
    }
    return REGK_OK;
}

int regk_reconcile(regk_ctx *ctx, const regk_decode_in *in, uint32_t flags, regk_delta *out)
{
    if (!ctx || !in || !out)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_reconcile: NULL argument");
    memset(out, 0, sizeof *out);
    return reconcile_run(ctx, in, nullptr, flags, out, nullptr, nullptr, "regk_reconcile");
}

int regk_reconcile_owned(regk_ctx *ctx, const regk_decode_in *in, const regk_node_stat *st, uint32_t flags, regk_delta_owned *out)
{
    if (!ctx || !in || !out)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_reconcile_owned: NULL argument");
    memset(out, 0, sizeof *out);
    ctx->rc_valid = false;
    if (!st)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_reconcile_owned: NULL stat; regk_reconcile compares bytes alone");
    if (st->zk_flags > 1u)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_reconcile_owned: zk_flags %u is not 0 (persistent) or 1 (EPHEMERAL); a "
                                               "sequential or container mode makes a path key meaningless", st->zk_flags);
    if (st->zk_flags == 1u && st->session == 0)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_reconcile_owned: EPHEMERAL nodes need the session id they are sent on");
    return reconcile_run(ctx, in, st, flags, &out->d, &out->replace, &out->n_replace, "regk_reconcile_owned");
}


int regk_reconcile_requests(regk_ctx *ctx, const regk_jute_opts *o, regk_frames *out)
{
    if (!ctx || !o || !out)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_reconcile_requests: NULL argument");
    memset(out, 0, sizeof *out);
    const bool replace = o->op == REGK_ZK_REPLACE, observed = o->flags & REGK_ZK_VERSION_OBSERVED;
    if (o->op != REGK_ZK_CREATE && o->op != REGK_ZK_DELETE && o->op != REGK_ZK_SETDATA && !replace)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_reconcile_requests: op %u is not create (1), delete (2), setData (5) or "
                                               "replace (256)", o->op);
    if (observed && o->op == REGK_ZK_CREATE)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_reconcile_requests: a CreateRequest carries no version to observe");
    if (o->group > 65536)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_reconcile_requests: at most 65536 operations per multi transaction");
    if (replace && o->group > 32768)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_reconcile_requests: at most 32768 replace entries (65536 operations) per "
                                               "multi transaction");
    if (ctx->pending)
        return fail(ctx, REGK_ERR_STATE, "regk_reconcile_requests: batches are still in flight; finish them first");
    if (!ctx->rc_valid)
        return fail(ctx, REGK_ERR_STATE, "regk_reconcile_requests: no reconcile result on this context; call regk_reconcile first");
    if ((replace || observed) && !ctx->rc_owned)
        return fail(ctx, REGK_ERR_STATE, "regk_reconcile_requests: replace frames and observed versions need node stats; the last "
                                         "reconcile was regk_reconcile, call regk_reconcile_owned");
    if (ctx->rc_owned && (replace || o->op == REGK_ZK_CREATE) && o->zk_flags != ctx->rc_zk_flags)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_reconcile_requests: zk_flags %u differs from the CreateMode %u regk_reconcile_owned "
                                               "classified with; nodes created so would be classed REPLACE again", o->zk_flags,
                    ctx->rc_zk_flags);
    CK(cudaSetDevice(ctx->device));
    /* gathered streams: create paths / payloads, update paths / payloads, delete paths, replace paths / payloads */
    const int g = o->op == REGK_ZK_CREATE ? RC_GCREATE : o->op == REGK_ZK_SETDATA ? RC_GUPDATE : replace ? RC_GREPLACE : RC_GDELETE;
    const int l = o->op == REGK_ZK_CREATE ? RC_LCREATE : o->op == REGK_ZK_SETDATA ? RC_LUPDATE : replace ? RC_LREPLACE : RC_LDELETE;
    const uint64_t c = ctx->rc_count[l];
    DevBuf *rb = ctx->rc;
    const bool data = g != RC_GDELETE;
    FrameSrc src{c, (const uint8_t *)rb[regk_ctx::RC_G0B + 2 * g].p, (const unsigned long long *)rb[regk_ctx::RC_G0B + 2 * g + 1].p,
                 data ? (const uint8_t *)rb[regk_ctx::RC_G0B + 2 * g + 2].p : nullptr,
                 data ? (const unsigned long long *)rb[regk_ctx::RC_G0B + 2 * g + 3].p : nullptr};
    src.who = "regk_reconcile_requests";
    if (!replace && !observed)
        return frame_requests(ctx, src, o, rb[regk_ctx::RC_FBYTES], rb[regk_ctx::RC_FOFF], ctx->h_rc_fbytes, ctx->h_rc_foff, out);
    const int v = l == RC_LUPDATE ? RC_VUPDATE : l == RC_LREPLACE ? RC_VREPLACE : RC_VDELETE;
    const int32_t *ver = observed ? (const int32_t *)rb[regk_ctx::RC_VER0 + v].p : nullptr;
    return frame_entry_requests(ctx, src, o, ver, replace, rb[regk_ctx::RC_FBYTES], rb[regk_ctx::RC_FOFF], ctx->h_rc_fbytes,
                                ctx->h_rc_foff, out);
}

static const char *reply_reason(uint32_t code)
{
    switch (code) {
    case RP_TRUNC: return "the stream ends inside the frame";
    case RP_BAD_LEN: return "a frame length below 16 (no room for a ReplyHeader)";
    case RP_NEG_XID: return "a negative xid other than -1 (notification) or -2 (ping)";
    case RP_XID_RANGE: return "an xid outside the framed requests";
    case RP_ERR_BODY: return "an error reply with a body";
    case RP_SUCC_LEN: return "a success frame whose length disagrees with its data length";
    case RP_NEG_DATA: return "a data length below -1";
    case RP_STAT_LEN: return "Stat.dataLength differs from the data the reply carries";
    case RP_ORDER: return "a reply out of order, or for a record that already has one";
    default: return "internal error";
    }
}

int regk_read_replies(regk_ctx *ctx, const uint8_t *bytes, uint64_t len, uint32_t flags, regk_replies *out)
{
    if (!ctx || !out)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_replies: NULL argument");
    memset(out, 0, sizeof *out);
    if (ctx->pending)
        return fail(ctx, REGK_ERR_STATE, "regk_read_replies: batches are still in flight; finish them first");
    if (!ctx->gd_valid)
        return fail(ctx, REGK_ERR_STATE, "regk_read_replies: no getData framing (regk_jute_requests with REGK_ZK_GETDATA) of the "
                                         "batch finished last");
    if (ctx->gd_gen != ctx->last_gen || !ctx->last_path_off)
        return fail(ctx, REGK_ERR_STATE, "regk_read_replies: a batch finished after the getData framing; frame its getData "
                                         "requests first");
    if (!bytes && len)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_replies: NULL stream of %llu bytes", (unsigned long long)len);
    const bool in_dev = flags & REGK_IN_DEVICE, dev_out = flags & REGK_OUT_DEVICE;
    if (in_dev && ((uintptr_t)bytes & 15u))
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_replies: misaligned device stream (16-byte alignment needed)");
    const uint64_t n = ctx->gd_n;
    const int32_t xb = ctx->gd_xid;
    for (int32_t reserved : {-1, -2})
        if ((uint64_t)((uint32_t)reserved - (uint32_t)xb) < n)
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_replies: the framed xids [%d, %d + %llu) cover %d, which ZooKeeper "
                                                   "uses for %s", xb, xb, (unsigned long long)n, reserved,
                        reserved == -1 ? "watch notifications" : "pings");
    if (n >= 0xFFFFFFFFull)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_replies: %llu records: must be below 2^32 - 1", (unsigned long long)n);
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    DevBuf *rb = ctx->rq;
    int rc;
    for (auto &ev : ctx->rq_ev)
        if (!ev)
            CK(cudaEventCreate(&ev));
    const uint8_t *ds = bytes;
    if (!in_dev) {
        if ((rc = ensure_dev(ctx, rb[regk_ctx::RQ_STREAM], len + 16)))
            return rc;
        if (len)
            CK(cudaMemcpyAsync(rb[regk_ctx::RQ_STREAM].p, bytes, len, cudaMemcpyHostToDevice, s));
        ds = (const uint8_t *)rb[regk_ctx::RQ_STREAM].p;
    }
    const uint64_t nblk = (len + 15) / 16, tiles_s = (nblk + RP_TILE - 1) / RP_TILE, tiles_r = (n + RP_TILE - 1) / RP_TILE;
    uint64_t slots = 1024;
    while (slots < 2 * n)
        slots <<= 1;
    /* two-level totals of the candidate pass (the chain and node passes get theirs once the candidates are counted) */
    const size_t totals_bytes = align16(tiles_s * 4) + (tiles_s / SUPER + 1) * 8;
    const size_t n8 = n * 8 + 16, n4 = n * 4 + 16;
    if ((rc = ensure_dev(ctx, rb[regk_ctx::RQ_WORD], nblk * 4 + 16)) || (rc = ensure_dev(ctx, rb[regk_ctx::RQ_TOTALS], totals_bytes)) ||
        (rc = ensure_dev(ctx, rb[regk_ctx::RQ_TBASE], tiles_s * 8 + 16)) || (rc = ensure_dev(ctx, rb[regk_ctx::RQ_ERRA], n4)) ||
        (rc = ensure_dev(ctx, rb[regk_ctx::RQ_DPOS], n8)) || (rc = ensure_dev(ctx, rb[regk_ctx::RQ_DLEN], n4)) ||
        (rc = ensure_dev(ctx, rb[regk_ctx::RQ_VER], n4)) || (rc = ensure_dev(ctx, rb[regk_ctx::RQ_OWN], n8)) ||
        (rc = ensure_dev(ctx, rb[regk_ctx::RQ_SLOT], n4)) || (rc = ensure_dev(ctx, rb[regk_ctx::RQ_TABLE], slots * 4)) ||
        (rc = ensure_dev(ctx, rb[regk_ctx::RQ_COUNT], RQ_NCOUNTERS * 8)) || (rc = ensure_host(ctx, ctx->h_rq_count, RQ_NCOUNTERS * 8)))
        return rc;
    RepParams p{};
    p.s = ds;
    p.len = len;
    p.xid_base = xb;
    p.n = n;
    p.word = (uint32_t *)rb[regk_ctx::RQ_WORD].p;
    p.tile_total = (uint32_t *)rb[regk_ctx::RQ_TOTALS].p;
    p.super_total = (unsigned long long *)((uint8_t *)rb[regk_ctx::RQ_TOTALS].p + align16(tiles_s * 4));
    p.tile_base = (unsigned long long *)rb[regk_ctx::RQ_TBASE].p;
    p.err = (int32_t *)rb[regk_ctx::RQ_ERRA].p;
    p.data_pos = (unsigned long long *)rb[regk_ctx::RQ_DPOS].p;
    p.dlen = (uint32_t *)rb[regk_ctx::RQ_DLEN].p;
    p.ver = (int32_t *)rb[regk_ctx::RQ_VER].p;
    p.own = (long long *)rb[regk_ctx::RQ_OWN].p;
    p.slot = (uint32_t *)rb[regk_ctx::RQ_SLOT].p;
    p.d_path = ctx->last_path_bytes;
    p.d_path_off = ctx->last_path_off;
    p.table = (uint32_t *)rb[regk_ctx::RQ_TABLE].p;
    p.mask_t = (uint32_t)(slots - 1);
    p.counters = (unsigned long long *)rb[regk_ctx::RQ_COUNT].p;
    unsigned long long *hc = (unsigned long long *)ctx->h_rq_count.p;
    CK(cudaMemsetAsync(p.counters, 0, RQ_NCOUNTERS * 8, s));
    CK(cudaMemsetAsync(p.counters + RQ_ERR, 0xFF, 8, s));
    CK(cudaMemsetAsync(p.tile_total, 0, totals_bytes, s));
    CK(cudaEventRecord(ctx->rq_ev[0], s));
    uint32_t launches = 0;
    /* 1. candidates: the plausible positions; their count from the CTA totals' upper level */
    const uint64_t nsup = tiles_s / SUPER + 1;
    std::vector<unsigned long long> sup(nsup, 0);
    if (len) {
        regk_replies_cand_kernel<<<(unsigned)tiles_s, RP_TILE, 0, s>>>(p);
        CK(cudaGetLastError());
        launches++;
        CK(cudaMemcpyAsync(sup.data(), p.super_total, nsup * 8, cudaMemcpyDeviceToHost, s));
    }
    cudaError_t e = cudaStreamSynchronize(s);
    if (e != cudaSuccess)
        return fail(ctx, REGK_ERR_CUDA, "regk_read_replies: kernel execution failed: %s", cudaGetErrorString(e));
    uint64_t C = 0;
    for (unsigned long long v : sup)
        C += v;
    if (C >= 0xFFFFFFFFull)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_replies: %llu plausible frame positions in the stream: must be below "
                                               "2^32 - 1", (unsigned long long)C);
    /* 2. positions, successors, the jump tables J_0 .. J_K (2^(K+1) >= C), the chain from position 0 */
    uint32_t K = 0;
    while ((1ull << (K + 1)) < C)
        K++;
    const size_t tiles_c = (C + RP_TILE - 1) / RP_TILE, tiles2 = std::max<uint64_t>(tiles_c, tiles_r);
    const size_t totals2_bytes = align16(tiles2 * 4) + (tiles2 / SUPER + 1) * 8;
    if ((rc = ensure_dev(ctx, rb[regk_ctx::RQ_CAND], C * 8 + 16)) || (rc = ensure_dev(ctx, rb[regk_ctx::RQ_MARK], C + 16)) ||
        (rc = ensure_dev(ctx, rb[regk_ctx::RQ_JUMP], (size_t)(K + 1) * C * 4 + 16)) ||
        (rc = ensure_dev(ctx, rb[regk_ctx::RQ_TOTALS2], totals2_bytes)))
        return rc;
    p.cand = (unsigned long long *)rb[regk_ctx::RQ_CAND].p;
    p.marked = (uint8_t *)rb[regk_ctx::RQ_MARK].p;
    p.C = C;
    uint32_t *J = (uint32_t *)rb[regk_ctx::RQ_JUMP].p;
    RepParams p2 = p;                                   /* the chain and node passes' totals */
    p2.tile_total = (uint32_t *)rb[regk_ctx::RQ_TOTALS2].p;
    p2.super_total = (unsigned long long *)((uint8_t *)rb[regk_ctx::RQ_TOTALS2].p + align16(tiles2 * 4));
    const unsigned g256 = (unsigned)((C + 255) / 256);
    if (C) {
        regk_replies_compact_kernel<<<(unsigned)tiles_s, RP_TILE, 0, s>>>(p);
        regk_replies_succ_kernel<<<g256, 256, 0, s>>>(p, J);
        for (uint32_t l = 0; l < K; l++)
            regk_replies_jump_kernel<<<g256, 256, 0, s>>>(J + (size_t)l * C, J + (size_t)(l + 1) * C, C);
        CK(cudaMemsetAsync(p.marked, 0, C, s));
        for (uint32_t l = K + 1; l-- > 0;)
            regk_replies_mark_kernel<<<g256, 256, 0, s>>>(p, J + (size_t)l * C, l == K ? 1u : 0u);
        /* 3. the chain's replies: k, the full check, the per-record arrays */
        CK(cudaMemsetAsync(p2.tile_total, 0, totals2_bytes, s));
        regk_replies_chain_count_kernel<<<(unsigned)tiles_c, RP_TILE, 0, s>>>(p2);
        regk_replies_chain_kernel<<<(unsigned)tiles_c, RP_TILE, 0, s>>>(p2);
        CK(cudaGetLastError());
        launches += 2 * K + 6;
    }
    CK(cudaMemcpyAsync(hc, p.counters, RQ_NCOUNTERS * 8, cudaMemcpyDeviceToHost, s));
    e = cudaStreamSynchronize(s);
    if (e != cudaSuccess)
        return fail(ctx, REGK_ERR_CUDA, "regk_read_replies: kernel execution failed: %s", cudaGetErrorString(e));
    if (hc[RQ_ERR] != ~0ull) {
        /* the smallest record whose frame fails the full check; the frame starts 24 bytes before its data */
        const uint64_t k = hc[RQ_ERR] >> 8;
        const uint32_t code = (uint32_t)(hc[RQ_ERR] & 0xFF);
        unsigned long long dpos = 0;
        CK(cudaMemcpyAsync(&dpos, p.data_pos + k, 8, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        const uint64_t pos = dpos - 24;
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_replies: byte %llu: %s; expected the reply to record %llu (xid %d)",
            (unsigned long long)pos, reply_reason(code), (unsigned long long)k, (int32_t)((uint32_t)xb + (uint32_t)k));
    }
    if (hc[RQ_NREP] < n) {
        /* the chain stops before the n-th reply: the full check where it stops names the reason */
        uint64_t stop = 0;
        if (C) {
            regk_replies_stop_kernel<<<g256, 256, 0, s>>>(p);
            CK(cudaGetLastError());
            CK(cudaMemcpyAsync(hc + RQ_STOP, p.counters + RQ_STOP, 8, cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
            stop = hc[RQ_STOP];
        }
        const uint64_t done = hc[RQ_NREP];
        uint8_t head[24] = {0};
        const uint64_t avail = len - stop, take = std::min<uint64_t>(avail, sizeof head);
        if (take) {
            CK(cudaMemcpyAsync(head, ds + stop, take, cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
        }
        ReplyHead h;
        const uint32_t code = reply_head(head, avail, xb, n, &h);
        const int32_t want = (int32_t)((uint32_t)xb + (uint32_t)done);
        if (code == RP_TRUNC)
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_replies: byte %llu: the stream ends before the reply to record %llu "
                                                   "(xid %d) is complete; %llu of %llu replies complete", (unsigned long long)stop,
                        (unsigned long long)done, want, (unsigned long long)done, (unsigned long long)n);
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_replies: byte %llu: %s (len %d, xid %d); expected the reply to record "
                                               "%llu (xid %d)", (unsigned long long)stop, code ? reply_reason(code) : "internal error",
                    h.len, h.xid, (unsigned long long)done, want);
    }
    /* 4. the nodes: found records, one per distinct path, in record order */
    if ((rc = ensure_dev(ctx, rb[regk_ctx::RQ_NREC], n8)) || (rc = ensure_dev(ctx, rb[regk_ctx::RQ_NVER], n4)) ||
        (rc = ensure_dev(ctx, rb[regk_ctx::RQ_NOWN], n8)) || (rc = ensure_dev(ctx, rb[regk_ctx::RQ_NPLEN], n4)) ||
        (rc = ensure_dev(ctx, rb[regk_ctx::RQ_NDLEN], n4)))
        return rc;
    p.node_rec = (unsigned long long *)rb[regk_ctx::RQ_NREC].p;
    p.node_ver = (int32_t *)rb[regk_ctx::RQ_NVER].p;
    p.node_own = (long long *)rb[regk_ctx::RQ_NOWN].p;
    p.node_plen = (uint32_t *)rb[regk_ctx::RQ_NPLEN].p;
    p.node_dlen = (uint32_t *)rb[regk_ctx::RQ_NDLEN].p;
    p.tile_total = p2.tile_total;
    p.super_total = p2.super_total;
    CK(cudaMemsetAsync(p.table, 0, slots * 4, s));
    CK(cudaMemsetAsync(p.tile_total, 0, totals2_bytes, s));
    regk_replies_insert_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(p);
    regk_replies_node_count_kernel<<<(unsigned)tiles_r, RP_TILE, 0, s>>>(p);
    regk_replies_node_kernel<<<(unsigned)tiles_r, RP_TILE, 0, s>>>(p);
    CK(cudaGetLastError());
    launches += 3;
    CK(cudaMemcpyAsync(hc, p.counters, RQ_NCOUNTERS * 8, cudaMemcpyDeviceToHost, s));
    e = cudaStreamSynchronize(s);
    if (e != cudaSuccess)
        return fail(ctx, REGK_ERR_CUDA, "regk_read_replies: kernel execution failed: %s", cudaGetErrorString(e));
    const uint64_t m = hc[RQ_M];
    /* 5. the snapshot's streams: node paths from the batch, node data from the reply stream */
    const uint64_t gt = (m + MK_TILE - 1) / MK_TILE;
    if ((rc = ensure_dev(ctx, rb[regk_ctx::RQ_GTOT], gt * 8 + (gt / SUPER + 1) * 8 + 16)) ||
        (rc = ensure_dev(ctx, rb[regk_ctx::RQ_PO], (m + 1) * 8)) || (rc = ensure_dev(ctx, rb[regk_ctx::RQ_JO], (m + 1) * 8)))
        return rc;
    uint64_t totals[2] = {0, 0};
    for (int g = 0; g < 2; g++) {
        DevBuf &gb = rb[g ? regk_ctx::RQ_JB : regk_ctx::RQ_PB], &go = rb[g ? regk_ctx::RQ_JO : regk_ctx::RQ_PO];
        MkGatherParams gp{};
        gp.n_dirs = m;
        gp.path_bytes = g ? ds : ctx->last_path_bytes;
        gp.path_off = g ? p.data_pos : ctx->last_path_off;
        gp.dir_rec = p.node_rec;
        gp.dir_len = g ? p.node_dlen : p.node_plen;
        gp.tile_total = (unsigned long long *)rb[regk_ctx::RQ_GTOT].p;
        gp.super_total = gp.tile_total + gt;
        gp.dir_off = (unsigned long long *)go.p;
        if (!m) {
            if ((rc = ensure_dev(ctx, gb, 16)))
                return rc;
            CK(cudaMemsetAsync(go.p, 0, 8, s));
            continue;
        }
        CK(cudaMemsetAsync(gp.super_total, 0, (gt / SUPER + 1) * 8, s));
        regk_mkdirp_len_kernel<<<(unsigned)gt, MK_TILE, 0, s>>>(gp);
        /* the stream's size: the sum of the upper level of the totals */
        std::vector<unsigned long long> gs(gt / SUPER + 1);
        CK(cudaMemcpyAsync(gs.data(), gp.super_total, gs.size() * 8, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        for (unsigned long long v : gs)
            totals[g] += v;
        if ((rc = ensure_dev(ctx, gb, totals[g] + 16)))
            return rc;
        gp.dir_bytes = (uint8_t *)gb.p;
        regk_mkdirp_gather_kernel<<<(unsigned)gt, MK_TILE, 0, s>>>(gp);
        CK(cudaGetLastError());
        launches += 2;
    }
    CK(cudaEventRecord(ctx->rq_ev[1], s));
    e = cudaStreamSynchronize(s);
    if (e != cudaSuccess)
        return fail(ctx, REGK_ERR_CUDA, "regk_read_replies: kernel execution failed: %s", cudaGetErrorString(e));
    float ms = 0;
    cudaEventElapsedTime(&ms, ctx->rq_ev[0], ctx->rq_ev[1]);
    const int32_t *err_out = p.err;
    const uint64_t *rec_out = (const uint64_t *)p.node_rec;
    if (!dev_out) {
        if ((rc = ensure_host(ctx, ctx->h_rq_err, n * 4 + 16)) || (rc = ensure_host(ctx, ctx->h_rq_node, m * 8 + 16)))
            return rc;
        if (n)
            CK(cudaMemcpyAsync(ctx->h_rq_err.p, p.err, n * 4, cudaMemcpyDeviceToHost, s));
        if (m)
            CK(cudaMemcpyAsync(ctx->h_rq_node.p, p.node_rec, m * 8, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        err_out = (const int32_t *)ctx->h_rq_err.p;
        rec_out = (const uint64_t *)ctx->h_rq_node.p;
    }
    out->n = n;
    out->m = m;
    out->n_found = hc[RQ_FOUND];
    out->n_missing = hc[RQ_MISSING];
    out->n_error = hc[RQ_ERROR];
    out->n_skipped = hc[RQ_SKIP];
    out->consumed = hc[RQ_CONSUMED];
    out->flags = dev_out ? REGK_OUT_DEVICE : 0;
    out->launches = launches;
    out->err = err_out;
    out->node_rec = rec_out;
    out->snapshot.n = m;
    out->snapshot.flags = REGK_IN_DEVICE;
    out->snapshot.path_total = totals[0];
    out->snapshot.json_total = totals[1];
    out->snapshot.path_bytes = (const uint8_t *)rb[regk_ctx::RQ_PB].p;
    out->snapshot.path_off = (const uint64_t *)rb[regk_ctx::RQ_PO].p;
    out->snapshot.json_bytes = (const uint8_t *)rb[regk_ctx::RQ_JB].p;
    out->snapshot.json_off = (const uint64_t *)rb[regk_ctx::RQ_JO].p;
    out->version = p.node_ver;
    out->ephemeral_owner = (const int64_t *)p.node_own;
    out->kernel_ms = ms;
    return REGK_OK;
}

int regk_release(regk_ctx *ctx, regk_result *res)
{
    if (!ctx || !res)
        return REGK_ERR_INVALID_ARG;
    /* single-slot ownership: buffers are recycled by the next batch; nothing to free eagerly */
    res->path_bytes = res->json_bytes = nullptr;
    res->path_off = res->json_off = nullptr;
    res->opaque = nullptr;
    return REGK_OK;
}

}  /* extern "C" */
