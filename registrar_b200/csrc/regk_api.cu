/*
 * regk_api.cu — C-ABI (include/regk.h) over the sm_90a kernels.
 *
 * Host-side plumbing only: argument checks, device buffers, the per-type JSON
 * fragment table, launch configuration, status read-back.  All record bytes
 * are produced by the kernels in regk_kernels.cuh; there is no CPU
 * implementation of the path in this library.
 */
#include <cuda_runtime.h>
#include <cub/device/device_radix_sort.cuh>

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <utility>
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
#include "regk_children.cuh"
#include "regk_results.cuh"
#include "regk_stats.cuh"
#include "regk_events.cuh"
#include "regk_setwatches.cuh"
#include "regk_resolve.cuh"
#include "regk_resolve_any.cuh"
#include "regk_dns.cuh"
#include "regk_dns_ptr.cuh"
#include "regk_walk.cuh"
#include "regk_walk_watch.cuh"
#include "regk_walk_setwatches.cuh"
#include "regk_walk_resolve.cuh"
#include "regk_types.hpp"

using namespace regk;

namespace {

thread_local std::string g_create_error;

/* Memory the context owns (ensure_dev / ensure_host grow it), freed with its owner. */
template <cudaError_t (*Free)(void *)>
struct Buf {
    void *p = nullptr;
    size_t cap = 0;
    Buf() = default;
    Buf(Buf &&o) noexcept : p(std::exchange(o.p, nullptr)), cap(std::exchange(o.cap, 0)) {}
    Buf &operator=(Buf &&o) noexcept
    {
        std::swap(p, o.p);
        std::swap(cap, o.cap);
        return *this;
    }
    ~Buf() { release(); }
    cudaError_t release()
    {
        const cudaError_t e = p ? Free(p) : cudaSuccess;
        p = nullptr;
        cap = 0;
        return e;
    }
};
using DevBuf = Buf<cudaFree>;
using HostBuf = Buf<cudaFreeHost>;

/* A CUDA event or stream the context owns, created on first use (ensure_event / ensure_stream). */
template <typename T, cudaError_t (*Destroy)(T)>
struct Handle {
    T h = nullptr;
    Handle() = default;
    Handle(Handle &&o) noexcept : h(std::exchange(o.h, nullptr)) {}
    Handle &operator=(Handle &&o) noexcept
    {
        std::swap(h, o.h);
        return *this;
    }
    ~Handle()
    {
        if (h)
            Destroy(h);
    }
    operator T() const { return h; }
};
using Event = Handle<cudaEvent_t, cudaEventDestroy>;
using Stream = Handle<cudaStream_t, cudaStreamDestroy>;

/* Request frames and their offsets, on the device and in pinned host memory (regk_frames). */
struct FrameBufs {
    DevBuf bytes, off;
    HostBuf h_bytes, h_off;
};

/* A parent pass (regk_parents.cuh): parent length and table slot per record, the table, tile totals, the distinct
   parents and their count. */
struct ParentPass {
    DevBuf len, slot, table, totals, unique;
};

}  // namespace

struct regk_ctx {
    ~regk_ctx();
    int device = 0;
    Stream own_stream;
    cudaStream_t stream = nullptr;              /* the stream work is enqueued on: own_stream or the caller's */
    std::string err;
    int sm_count = 0;
    int max_smem_optin = 0;
    /* compose kernels' L2 lookahead: CTAs of one wave by dynamic shared memory (lookahead_tiles); 0 alias paths,
       1 node paths, 2 payloads */
    std::map<size_t, uint32_t> wave_ctas[3];

    /* type table */
    std::vector<std::string> types;             /* raw */
    std::vector<uint8_t> blob_host;             /* TypeFrag[] + fragments, padded to 16 */
    DevBuf blob_dev;
    uint32_t max_type_q = 0;                    /* longest escaped type */

    /* A batch's device staging of host inputs, device outputs and pinned results.  sync_set serves every batch but
       "async" host batches (a job step uses none of it: its inputs and outputs are the caller's); the skip-mode redo
       and regk_service_records write into its device outputs too.  "async" host batches alternate between the two of hset: batch
       k+1's H2D and kernels overlap batch k's D2H (issued when k+1 is submitted or k is finished, whichever comes
       first - the copy sizes are only known once k's kernels are done). */
    struct HostSet {
        DevBuf in[11];
        DevBuf path_bytes, path_off, json_bytes, json_off, off32_p, off32_j;
        HostBuf h_path_bytes, h_path_off, h_json_bytes, h_json_off;
        Event e_in, e_out;                      /* async sets: staging copied in, results copied out */
    };
    HostSet sync_set, hset[2];
    uint64_t hseq = 0;
    bool is_async(const HostSet *hs) const { return hs != &sync_set; }
    HostBuf h_running;                          /* run_pipelined: each chunk's running payload total */
    Stream s_h2d, s_d2h;                        /* host pipelining (run_pipelined, two-deep async) */
    HostBuf h_gather_flag;                      /* uint32: 1 = regk_gather_push found the whole-job buffers too small,
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
    HostBuf h_job_bases;                        /* pinned copies of job_bases, NSLOTS * 8 entries */
    /* the device streams of the batch finished last: regk_parent_dirs, regk_mkdirp_dirs, regk_jute_requests,
       regk_decode, the reconcile calls and regk_read_replies work on them; written by set_last only */
    struct LastBatch {
        const uint8_t *path_bytes = nullptr;
        const unsigned long long *path_off = nullptr;
        uint64_t n = 0;                         /* records of the path stream, 0 without one */
        const uint8_t *json_bytes = nullptr;
        const unsigned long long *json_off = nullptr;
        uint64_t json_n = 0;                    /* ... and of the payload stream */
        const uint32_t *host_off = nullptr;     /* how its paths end: hostname lengths (NULL: fixed stride) */
        uint32_t host_stride = 0;
        bool alias = false;
        uint64_t gen = 0;                       /* bumped whenever the fields above change */
    } last;
    FrameBufs frames;                           /* regk_jute_requests */
    /* regk_decode: staged streams, records, domain image and ports */
    struct Decode {
        DevBuf in[4], rec, dom, ports;
        HostBuf h_rec, h_dom, h_ports;
    } dec;
    /* regk_service_records: staged inputs, status + tile totals (the framing calls borrow it for their status) */
    struct Service {
        DevBuf in[7], work;
    } svc;
    /* regk_parent_dirs */
    struct Parents {
        ParentPass pass;
        HostBuf h_len, h_unique, h_count;
        Event ev[2];
    } par;
    /* regk_mkdirp_dirs (regk_mkdirp.cuh): its own parent pass, work lists, table, the set; regk_mkdirp_requests */
    struct Mkdirp {
        ParentPass pass;
        DevBuf flags, list[2], totals, table, count, drec, dlen, dbytes, doff, depth, invalid, zero;
        HostBuf h_count, h_drec, h_dlen, h_dbytes, h_doff, h_depth, h_invalid;
        Event ev[4];
        FrameBufs frames;
        bool valid = false;                     /* the set of the last regk_mkdirp_dirs call is in drec .. invalid */
        uint64_t n_dirs = 0, bytes = 0;
        uint64_t gen = 0;                       /* bumped by every regk_mkdirp_dirs */
    } mk;
    /* regk_reconcile / regk_reconcile_owned (regk_reconcile.cuh): staged snapshot and stats, tables, outputs, lists,
       versions, the gathered request streams; regk_reconcile_requests' frames */
    struct Reconcile {
        DevBuf in[6];                           /* path bytes, path offsets, data bytes, data offsets, versions, owners */
        DevBuf t_obs, t_des, slot_obs, hash_obs, slot_des, cls, match, obs_cls, totals, count, gtotals;
        DevBuf list[RC_NLISTS], len[RC_NGATHERS], ver[RC_NVER];
        struct {
            DevBuf bytes, off;
        } gather[RC_NGATHERS];
        HostBuf h_count, h_cls, h_match, h_obs_cls, h_list[RC_NLISTS];
        Event ev[2];
        FrameBufs frames;
        bool valid = false;                     /* the request streams of the last reconcile call are in gather */
        bool owned = false;                     /* ... and it was regk_reconcile_owned: versions in ver */
        uint32_t zk_flags = 0;                  /* the CreateMode regk_reconcile_owned classified with */
        uint64_t n_list[RC_NLISTS] = {};        /* entries of each list: create, update, dup, replace, delete */
        uint64_t gen = 0;                       /* bumped by every reconcile call */
    } rc;
    /* the last REGK_ZK_GETDATA framing: the batch it framed, xid_base, n (regk_read_replies reads its replies) */
    bool gd_valid = false;
    uint64_t gd_gen = 0, gd_n = 0;
    int32_t gd_xid = 0;
    /* regk_read_replies (regk_replies.cuh): staged stream, candidates, jump tables, per-record arrays, table, the nodes
       and the gathered snapshot */
    struct Replies {
        DevBuf stream, word, totals, totals2, tile_base, cand, mark, jump, err, data_pos, dlen, ver, own, slot, table;
        DevBuf node_rec, node_ver, node_own, node_plen, node_dlen, gtotals, count;
        DevBuf snap_bytes[2], snap_off[2];      /* the snapshot's path and data streams */
        HostBuf h_count, h_err, h_node;
        Event ev[2];
    } rq;
    /* regk_children_requests / regk_read_children (regk_children.cuh).  The last REGK_ZK_GETCHILDREN framing: its own
       parent pass, the directory set (listed and unlisted) and its packed bytes, the batch it framed, xid_base, d.
       The last read: frame and entry chains, per-directory arrays, the listing, the keep table, the stale list and
       its packed paths (the REGK_ZK_DELETE framing reads those), and copies of the set it read against. */
    struct Children {
        ParentPass pass;
        DevBuf totals, count, unlisted, drec, dlen, dbytes, doff;
        HostBuf h_count;
        FrameBufs frames[2];                    /* getChildren, delete */
        bool framed = false;
        uint64_t gen = 0, n = 0, d = 0, n_unlisted = 0, prefixes = 0;
        int32_t xid = 0;
        DevBuf stream, word, ftotals, tile_base, cand, mark, jump, totals2, fpos, fend, err, cnt, seed_g, last_g1, name_bad,
            end_pos, fault_pos, child_off;
        DevBuf eword, etotals, etile_base, ecand, emark, ejump, etotals2, ent_pos, ent_nlen, ent_k, ent_plen;
        DevBuf gtotals, lst_bytes, lst_off, lst_zero, table, cls, stotals, stale, stale_len, sbytes, soff;
        DevBuf r_drec, r_dlen, r_unlisted;
        HostBuf h_drec, h_dlen, h_err, h_child_off, h_cls, h_stale, h_unlisted;
        Event ev[2];
        bool read = false;                      /* the stale list of the last regk_read_children is in stale .. soff */
        uint64_t n_stale = 0;
        uint64_t read_gen = 0;                  /* bumped by every regk_read_children */
        /* the directories whose prefixes go into the keep table: the framed ones, or the batch's whole set when
           regk_events_requests framed a subset of it */
        const unsigned long long *keep_drec = nullptr;
        const uint32_t *keep_dlen = nullptr;
        uint64_t keep_d = 0;
        /* a subset framing of regk_events_requests: directory k of the framing is directory sub_item[k] of the batch's
           whole set (NULL: the framing lists the whole set) */
        const unsigned long long *sub_item = nullptr;
    } ch;
    /* regk_read_results (regk_results.cuh): what each write framing framed (one record per source, four for the
       reconcile ops), and the last read's chain, per-frame and per-entry arrays and lists */
    struct ResDesc {
        bool valid = false;
        ResFraming f{};
        const unsigned long long *subject = nullptr;    /* device: what entry e stands for; NULL = e */
        int32_t tol = 0;                        /* the code that still counts as done */
        uint64_t gen = 0;                       /* the generation of the state it framed */
    };
    struct Results {
        ResDesc batch, mkdirp, stale, rec[4];   /* rec: create, delete, setData, replace */
        DevBuf stream, word, totals, tile_base, cand, mark, jump, totals2, count, fpos, ferr, err, cls, ver, subject, fault_at,
            ltotals, failed, aborted;
        HostBuf h_count, h_ferr, h_err, h_cls, h_ver, h_subject, h_failed, h_aborted;
        Event ev[2];
    } rs;
    /* the last REGK_ZK_EXISTS framing (as gd_* above), and regk_read_stats (regk_stats.cuh): staged stream, candidates,
       jump tables, the per-record arrays regk_reconcile_stats classes from, and the batch they answer */
    bool ex_valid = false;
    uint64_t ex_gen = 0, ex_n = 0;
    int32_t ex_xid = 0;
    struct Stats {
        DevBuf stream, word, totals, tile_base, cand, mark, jump, totals2, count, fpos, err, ver, own, dlen, mzxid, known;
        HostBuf h_count, h_err, h_ver, h_own, h_dlen, h_mzxid;
        Event ev[2];
        bool read = false;                      /* the arrays of the last regk_read_stats are in err .. mzxid */
        uint64_t gen = 0, n = 0;                /* the batch generation and the records they answer */
        /* a subset read (regk_events_requests): record k of the arrays is sub_rec[k] of a batch of batch_n records;
           regk_reconcile_stats spreads it over f_err .. f_dlen */
        bool sub = false;
        uint64_t batch_n = 0;
        DevBuf sub_rec, f_err, f_ver, f_own, f_dlen;
    } sq;
    /* the subset of the last REGK_ZK_EXISTS framing of regk_events_requests (ex_sub; ex_n records, listed in ex_rec) */
    bool ex_sub = false;
    const unsigned long long *ex_rec = nullptr;
    /* regk_read_events / regk_events_requests (regk_events.cuh).  Per batch generation: the directory set (the members
       children_dirs fills), the record and directory tables, the marks and the pending counts.  Per call: the staged
       stream, the chain, the events.  Per framing: the pending set compacted and its packed paths. */
    struct Events {
        ParentPass pass;
        DevBuf totals, count, unlisted, drec, dlen, dbytes, doff;
        HostBuf h_count;
        uint64_t d = 0, n_unlisted = 0, prefixes = 0;
        bool built = false, read = false;       /* tables of batch generation `gen`; events read for it */
        uint64_t gen = 0, n = 0;
        uint32_t rec_epoch = 1, dir_epoch = 1, mask_r = 0, mask_d = 0;
        DevBuf zero, slot, t_rec, t_dir, rec_mark, dir_mark, dirty;
        DevBuf stream, word, ftotals, tile_base, cand, mark, jump, ntotals, ecount;
        DevBuf pos, type, state, zxid, kind, subject;
        HostBuf h_ecount, h_pos, h_type, h_state, h_zxid, h_kind, h_subject;
        Event ev[2];
        DevBuf ptotals, pcount, item[2], prec[2], plen[2], pbytes, poff;
        FrameBufs frames;
    } evq;
    /* the watches the session holds (regk_setwatches.cuh), for batch generation `gen`: the kind each watched read armed
       per record and per directory of evq's set, whether the last exists / getChildren framing carried the watch byte
       and whether its replies are still unread (in flight), and regk_read_events' SetWatches gate.  zxid: the session's
       high-water mark, kept for the context's whole life.  The framing's working arrays and frames. */
    struct Watch {
        uint64_t gen = 0;
        DevBuf rec_kind, dir_kind;
        uint64_t rec_n = 0, dir_d = 0;          /* kinds held for this generation; 0: none yet (all NONE) */
        bool ex_watch = false, ch_watch = false;
        bool ex_fly = false, ch_fly = false;
        bool gate = false;
        bool lmax_ok = false;
        uint32_t lmax = 0;                      /* the batch's longest path */
        long long zxid = 0;
        DevBuf zmax, lmax_d, cls, totals, count, ent_src, ent_s, ent_len;
        FrameBufs frames;
        Event ev[2];
    } wq;
    /* regk_resolve (regk_resolve.cuh): staged snapshot, table, decode outputs, per-node and per-child arrays, sort
       buffers, totals, the answers and their pinned copies */
    struct Resolve {
        DevBuf in[4], table, slot, hash, rec, dom, ports, cls, roles, ttl, key, val, skey, sval, first, end, cum[3], totals,
            count, node_q, q_kind, q_node, sec_off, unres, text, sort_tmp;
        DevBuf any_list, any_totals, any_count;     /* REGK_RESOLVE_ANY_FORM: the candidates, their tile totals, count */
        HostBuf h_count, h_q_kind, h_q_node, h_sec_off, h_text, h_cls, h_unres, h_any;
        Event ev[5];
        /* the last call succeeded: regk_dns_answer answers against it (the snapshot streams it read, its table size) */
        bool valid = false;
        bool walk = false;                      /* it was a regk_walk_resolve, of walk snapshot generation walk_sgen */
        uint64_t walk_sgen = 0;
        uint64_t gen = 0, m = 0, path_total = 0, slots = 0;
        const uint8_t *pb = nullptr, *jb = nullptr;
        const uint64_t *po = nullptr, *jo = nullptr;
    } rsv;
    /* regk_dns_answer (regk_dns.cuh): the per-resolve preparation (of resolve generation prep_gen), the staged queries,
       the per-query arrays and the responses.  REGK_DNS_PTR (regk_dns_ptr.cuh): the reverse index of resolve generation
       ptr_gen (0: not built), its n host nodes, the sort's inputs and temporary storage, its tile totals */
    struct Dns {
        uint64_t prep_gen = 0, ptr_gen = 0, ptr_n = 0;
        DevBuf ip4, cum[3], ptotals, in[2], scratch, status, tc, node, meta, nans, nadd, ans_bytes, qtotals, resp_off, rr_base,
            count, resp;
        DevBuf pkey_in, pval_in, pkey, pval, pbytes, ptr_tmp, ptr_totals, ptr_count;
        HostBuf h_count, h_resp_off, h_resp, h_status, h_tc, h_node;
        Event ev[4];
    } dns;
    /* regk_walk_start / regk_walk_requests / regk_read_walk (regk_walk.cuh): the frontier (packed paths from 0, their
       lengths; two sets, the next level is read into the other), the framing, the snapshot so far (grown
       geometrically, [0, cap) of each stream allocated), and the read's own chains, per-node arrays and level streams */
    struct Walk {
        bool active = false, framed = false;
        int cur = 0;
        uint64_t f = 0, fpt = 0;                /* nodes of the current frontier, their path bytes */
        DevBuf fbytes[2], foff[2], flen[2];
        int32_t xid = 0;
        FrameBufs frames;
        uint64_t m = 0, path_total = 0, data_total = 0;
        DevBuf snap_bytes[2], snap_off[2], ver, own;
        std::vector<uint64_t> level_off;
        DevBuf stream, word, totals, totals2, tile_base, cand, mark, jump, err, data_pos, dlen, dver, down, count;
        DevBuf cword, ctotals, ctile_base, ccand, cmark, cjump, ctotals2, fpos, fend, cerr, cnt, seed_g, last_g1, name_bad,
            end_pos, fault_pos, child_off, eword, etotals, etile_base, ecand, emark, ejump, etotals2, ent_pos, ent_nlen, ent_k;
        DevBuf ftotals, node_rec, node_ver, node_own, node_plen, node_dlen, wcount, gtotals, lvl_bytes[2], lvl_off[2];
        HostBuf h_count, h_wcount;
        Event ev[2];
        /* watches (regk_walk_watch.cuh).  watched: every level read was framed with REGK_ZK_WATCH (framed_watch: the
           current framing was); refreshed: a regk_walk_refresh ran since the start (listings are then filtered);
           rlevel: the frontier is a refresh level, frontier node i being snapshot node fnode[i].  The marks and their
           counts (mcount: pending, removed) per node; the path table holds nodes [0, tab_m) and is valid while
           tab_rgen == rgen (rgen counts the rebuilds, which renumber the nodes).  The rebuild writes the other set of
           snapshot arrays and swaps. */
        bool watched = true, framed_watch = false, refreshed = false, rlevel = false, tab_valid = false;
        uint64_t rgen = 0, tab_rgen = 0, tab_m = 0, n_pending = 0, n_removed = 0;
        uint32_t tab_mask = 0;
        DevBuf wmark, mcount, table, fnode, rpos, rlen, snap2_bytes[2], snap2_off[2], ver2, own2, wmark2;
        DevBuf ktotals, kcount, psrc, dsrc, kplen, kdlen, dsel, xkeep, xtotals, xrec, xlen, xcount, xbytes, xoff;
        DevBuf vstream, vword, vtotals, vtile_base, vcand, vmark, vjump, vcount, vntotals, e_pos, e_type, e_state, e_zxid,
            e_node, e_parent;
        HostBuf h_epos, h_etype, h_estate, h_ezxid, h_enode, h_vcount;
        Event eev[4];
        /* across a reconnect (regk_walk_setwatches.cuh): the armed byte per node (armed2: the rebuild's copy), the
           walk's zxid high-water mark (largest ReplyHeader.zxid of the replies its successful reads and event calls
           walked), the SetWatches gate of regk_walk_events, and the framing's working arrays and frames */
        DevBuf armed, armed2, zmax, sw_lmax, sw_cls, sw_totals, sw_count, sw_ent_src, sw_ent_s, sw_ent_len;
        long long zxid = 0;
        bool gate = false;
        FrameBufs swframes;
        Event swev[2];
        /* regk_walk_resolve (regk_walk_resolve.cuh): the identity word per node (ident2: the rebuild's copy), and the
           snapshot generation, bumped whenever the snapshot's nodes or buffers change (regk_dns_answer's gate) */
        DevBuf ident, ident2;
        uint64_t sgen = 0;
    } wk;
    /* regk_walk_resolve: the last successful call (have; its default TTLs) and its text and run offsets (set cur; the
       other set is written by the next call and becomes cur on success), the pieces and segments of one call */
    struct WalkResolve {
        bool have = false;
        int cur = 0;
        int32_t dflt_host = 0, dflt_srv = 0;
        bool any = false;                       /* the last call's REGK_RESOLVE_ANY_FORM */
        uint64_t segments = 0;
        DevBuf text[2], run[2], kind, len, src, dest, totals, count, seg_src, seg_dest, seg_sel, seg_len, seg_off, scratch;
        Event ev[4];
    } wr;
    std::vector<Event> pipe_events;             /* run_pipelined */
    /* skip mode (regk_skip.cuh): fence workspace, the compacted batch, the expanded offsets, the skipped list */
    struct Skip {
        DevBuf work, in[11], off_p, off_j, index, bits;
        HostBuf h_status, h_index, h_bits;
        struct Last {
            bool valid = false;                 /* the batch finished last was a skip-mode batch */
            uint64_t n = 0, n_skipped = 0;
            uint32_t bad_bits = 0;
        } last;
    } skip;
    /* workspace: DevStatus | two-level byte totals of both halves (stream-ordered reuse; host pipelining) */
    DevBuf work;
    /* device-resident batches rotate through a ring of workspaces that a side stream re-zeroes (and copies
       the status out of) after each use, so the main stream carries nothing but the two kernels */
    static constexpr int NWORK = 4;
    DevBuf work_ring[NWORK];
    Event ws_clean[NWORK];
    size_t ws_clean_bytes[NWORK] = {0, 0, 0, 0};
    Stream s_side;
    uint64_t ws_seq = 0;

    /* in-flight batches: events + pinned status per slot.  Outputs are single-buffered: with the
       "async" option several batches may be enqueued back to back (benchmark loops), each one
       overwriting the previous batch's outputs in stream order. */
    struct Slot {
        Event ev[6];                            /* [5]: after a job step's closing exchange */
        PathParams path_params{};               /* kept for the exact-offset redo (empty labels) */
        size_t path_smem = 0;
        bool path_alias = false, did_path = false;
        DevStatus *d_status = nullptr;
        DevStatus *h_status = nullptr;          /* pinned */
        int ring = -1;                          /* workspace ring entry used by this batch */
        HostSet *set = nullptr;                 /* where its staging, outputs and host results live */
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
    HostBuf h_status_block;                     /* DevStatus[NSLOTS] */
    uint64_t seq = 0;
    int pending = 0;

    std::map<std::string, int64_t> opt;
};

/* Work still enqueued on the context's streams may use its memory: wait for it before the members go.  Errors are
   ignored - this also runs at interpreter exit, while the CUDA runtime unloads.  A caller's stream is waited for,
   never destroyed. */
regk_ctx::~regk_ctx()
{
    cudaSetDevice(device);
    for (cudaStream_t s : {stream, (cudaStream_t)s_h2d, (cudaStream_t)s_d2h, (cudaStream_t)s_side})
        if (s)
            cudaStreamSynchronize(s);
}

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
    CK(b.release());
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
    CK(b.release());
    cudaError_t e = cudaMallocHost(&b.p, bytes);
    if (e != cudaSuccess)
        return fail(ctx, REGK_ERR_NOMEM, "cudaMallocHost(%zu) failed: %s", bytes, cudaGetErrorString(e));
    b.cap = bytes;
    return REGK_OK;
}

int ensure_event(regk_ctx *ctx, Event &ev, unsigned flags = cudaEventDefault)
{
    if (!ev.h)
        CK(cudaEventCreateWithFlags(&ev.h, flags));
    return REGK_OK;
}

int ensure_stream(regk_ctx *ctx, Stream &s)
{
    if (!s.h)
        CK(cudaStreamCreateWithFlags(&s.h, cudaStreamNonBlocking));
    return REGK_OK;
}

/* `bytes` of a host array into `b` (grown to bytes + 16), enqueued on s */
int stage_in(regk_ctx *ctx, DevBuf &b, const void *host, size_t bytes, cudaStream_t s)
{
    const int rc = ensure_dev(ctx, b, bytes + 16);
    if (rc)
        return rc;
    if (bytes)
        CK(cudaMemcpyAsync(b.p, host, bytes, cudaMemcpyHostToDevice, s));
    return REGK_OK;
}

/* `bytes` of device memory into the pinned buffer `b` (grown to bytes + 16), enqueued on s */
int to_host(regk_ctx *ctx, HostBuf &b, const void *dev, size_t bytes, cudaStream_t s)
{
    const int rc = ensure_host(ctx, b, bytes + 16);
    if (rc)
        return rc;
    if (bytes)
        CK(cudaMemcpyAsync(b.p, dev, bytes, cudaMemcpyDeviceToHost, s));
    return REGK_OK;
}

/* wait for the work enqueued on s; a fault fails the call as "<who>: kernel execution failed" */
int sync_or_fail(regk_ctx *ctx, cudaStream_t s, const char *who)
{
    const cudaError_t e = cudaStreamSynchronize(s);
    if (e != cudaSuccess)
        return fail(ctx, REGK_ERR_CUDA, "%s: kernel execution failed: %s", who, cudaGetErrorString(e));
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

/* cudaFuncAttributeMaxDynamicSharedMemorySize is per function and device, shared by every context of the process:
   raise it monotonically, and only when it grows (setting it is not free) */
int set_smem_limit(regk_ctx *ctx, const void *kernel, size_t bytes)
{
    static std::mutex mu;
    static std::map<std::pair<int, const void *>, size_t> high;
    std::lock_guard<std::mutex> lock(mu);
    size_t &h = high[{ctx->device, kernel}];
    if (bytes <= h)
        return REGK_OK;
    CK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    h = bytes;
    return REGK_OK;
}

/* The batch finished last is now the one whose device streams are given (NULL: not produced); n is its size. */
void set_last(regk_ctx *ctx, const uint8_t *path_bytes, const unsigned long long *path_off, const uint8_t *json_bytes,
    const unsigned long long *json_off, uint64_t n, const uint32_t *host_off, uint32_t host_stride, bool alias)
{
    ctx->last = {path_bytes, path_off, path_off ? n : 0, json_bytes, json_off, json_off ? n : 0, host_off, host_stride, alias,
                 ctx->last.gen + 1};
}

/* the pinned flag of regk_gather_push and the job exchanges, zeroed when first made */
int ensure_gather_flag(regk_ctx *ctx)
{
    if (ctx->h_gather_flag.p)
        return REGK_OK;
    const int rc = ensure_host(ctx, ctx->h_gather_flag, sizeof(uint32_t));
    if (rc == REGK_OK)
        *(uint32_t *)ctx->h_gather_flag.p = 0;
    return rc;
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

static int run_pipelined(regk_ctx *ctx, regk_ctx::HostSet &hs, const regk_batch *b, regk_result *res, const PathParams &pp0,
    size_t path_smem, const JsonParams &jp0, size_t json_smem, const HostPipe &hp)
{
    const uint64_t n = b->n;
    const bool alias = b->flags & REGK_NODE_ALIAS;
    const bool do_path = !(b->flags & REGK_NO_PATH), do_json = !(b->flags & REGK_NO_JSON);
    const uint32_t stride = b->host_stride;
    cudaStream_t s = ctx->stream;
    int rc;
    if ((rc = ensure_stream(ctx, ctx->s_h2d)) || (rc = ensure_stream(ctx, ctx->s_d2h)))
        return rc;
    ctx->pipe_events.resize(std::max<size_t>(ctx->pipe_events.size(), 3 * hp.nchunks + 2));
    for (Event &ev : ctx->pipe_events)
        if ((rc = ensure_event(ctx, ev, cudaEventDisableTiming)))
            return rc;
    if ((rc = ensure_host(ctx, hs.h_path_bytes, hp.path_cap)) || (rc = ensure_host(ctx, hs.h_path_off, (n + 1) * 8)) ||
        (rc = ensure_host(ctx, hs.h_json_bytes, hp.json_cap)) || (rc = ensure_host(ctx, hs.h_json_off, (n + 1) * 8)) ||
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
                CK(cudaMemcpyAsync((uint8_t *)hs.h_path_bytes.p + lo, (uint8_t *)hs.path_bytes.p + lo, hi - lo,
                    cudaMemcpyDeviceToHost, ctx->s_d2h));
            CK(cudaMemcpyAsync((uint64_t *)hs.h_path_off.p + r0, (uint64_t *)hs.path_off.p + r0, (r1 - r0 + (last ? 1 : 0)) * 8,
                cudaMemcpyDeviceToHost, ctx->s_d2h));
        }
        if (do_json) {
            const uint64_t lo = h_running[c], hi = std::min<uint64_t>(h_running[c + 1], hp.json_cap);
            if (hi > lo)
                CK(cudaMemcpyAsync((uint8_t *)hs.h_json_bytes.p + lo, (uint8_t *)hs.json_bytes.p + lo, hi - lo,
                    cudaMemcpyDeviceToHost, ctx->s_d2h));
            CK(cudaMemcpyAsync((uint64_t *)hs.h_json_off.p + r0, (uint64_t *)hs.json_off.p + r0, (r1 - r0 + (last ? 1 : 0)) * 8,
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
    res->path_bytes = (uint8_t *)hs.h_path_bytes.p;
    res->path_off = (uint64_t *)hs.h_path_off.p;
    res->json_bytes = (uint8_t *)hs.h_json_bytes.p;
    res->json_off = (uint64_t *)hs.h_json_off.p;
    if (!do_path)
        memset(res->path_off, 0, (n + 1) * 8);
    if (!do_json)
        memset(res->json_off, 0, (n + 1) * 8);
    return REGK_OK;
}

/* D2H of a host batch's results into its set's pinned buffers, enqueued on sd once the batch's status has reached the
   host (its kernels are done), so the exact byte counts are known. */
static int enqueue_d2h(regk_ctx *ctx, regk_ctx::Slot &slot, cudaStream_t sd)
{
    const DevStatus st = *slot.h_status;
    regk_ctx::HostSet &hs = *slot.set;
    const uint64_t n = slot.n;
    const bool do_path = !(slot.flags & REGK_NO_PATH), do_json = !(slot.flags & REGK_NO_JSON);
    int rc;
    if ((rc = ensure_host(ctx, hs.h_path_bytes, st.path_total + 16)) || (rc = ensure_host(ctx, hs.h_path_off, (n + 1) * 8)) ||
        (rc = ensure_host(ctx, hs.h_json_bytes, st.json_total + 16)) || (rc = ensure_host(ctx, hs.h_json_off, (n + 1) * 8)))
        return rc;
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
    return REGK_OK;
}

/* The D2H of an async host batch, on the D2H stream; a batch that failed the fence or still needs the exact-offset
   redo is left to regk_finish. */
static int issue_d2h(regk_ctx *ctx, regk_ctx::Slot &slot)
{
    const DevStatus st = *slot.h_status;
    if (st.bad_bits || st.overflow)
        return REGK_OK;
    if (st.needs_exact && slot.did_path)
        return REGK_OK;
    const int rc = enqueue_d2h(ctx, slot, ctx->s_d2h);
    if (rc)
        return rc;
    CK(cudaEventRecord(slot.set->e_out, ctx->s_d2h));
    slot.d2h_issued = true;
    return REGK_OK;
}

/* a host batch's results as regk_finish hands them out: the pinned buffers of its set */
static void host_results(regk_result *res, const regk_ctx::HostSet &hs, bool off32)
{
    res->flags = 0;
    res->path_bytes = (uint8_t *)hs.h_path_bytes.p;
    res->json_bytes = (uint8_t *)hs.h_json_bytes.p;
    if (off32) {
        res->path_off32 = (uint32_t *)hs.h_path_off.p;
        res->json_off32 = (uint32_t *)hs.h_json_off.p;
    } else {
        res->path_off = (uint64_t *)hs.h_path_off.p;
        res->json_off = (uint64_t *)hs.h_json_off.p;
    }
}

template <bool MULTI, bool DATA>
static int launch_jute(regk_ctx *ctx, const JuteParams &p, size_t smem)
{
    const int rc = set_smem_limit(ctx, (const void *)regk_jute_kernel<MULTI, DATA>, smem);
    if (rc)
        return rc;
    regk_jute_kernel<MULTI, DATA><<<(unsigned)((p.n + JUTE_TILE - 1) / JUTE_TILE), JUTE_THREADS, smem, ctx->stream>>>(p);
    CK(cudaGetLastError());
    return REGK_OK;
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
    uint32_t path_times, size_t slot_bytes, FrameBufs &fb, regk_frames *out, const std::function<int(const FrameGeom &)> &launch)
{
    DevBuf &db = fb.bytes, &doff = fb.off;
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
    if ((rc = ensure_dev(ctx, ctx->svc.work, 256)))
        return rc;
    CK(cudaMemsetAsync(ctx->svc.work.p, 0, sizeof(DevStatus), s));
    if (n == 0)
        CK(cudaMemsetAsync(doff.p, 0, 8, s));
    cudaEvent_t e0 = ctx->slots[0].ev[0], e1 = ctx->slots[0].ev[1];
    if (n) {
        FrameGeom g{};
        g.n = n;
        g.total = total;
        g.out_bytes = (uint8_t *)db.p;
        g.out_off = (unsigned long long *)doff.p;
        g.status = (DevStatus *)ctx->svc.work.p;
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
        if ((rc = launch(g)))
            return rc;
        CK(cudaEventRecord(e1, s));
        out->launches = 1;
    }
    CK(cudaMemcpyAsync(ctx->slots[0].h_status, ctx->svc.work.p, sizeof(DevStatus), cudaMemcpyDeviceToHost, s));
    if ((rc = sync_or_fail(ctx, s, src.who)))
        return rc;
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
    if ((rc = to_host(ctx, fb.h_bytes, db.p, total, s)) || (rc = to_host(ctx, fb.h_off, doff.p, (frames + 1) * 8, s)))
        return rc;
    CK(cudaStreamSynchronize(s));
    out->frame_bytes = (const uint8_t *)fb.h_bytes.p;
    out->frame_off = (const uint64_t *)fb.h_off.p;
    return REGK_OK;
}

static int frame_requests(regk_ctx *ctx, const FrameSrc &src, const regk_jute_opts *o, FrameBufs &fb, regk_frames *out)
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
    if (o->op == REGK_ZK_GETDATA || o->op == REGK_ZK_GETCHILDREN || o->op == REGK_ZK_EXISTS) {
        tail[0] = (o->flags & REGK_ZK_WATCH) ? 1u : 0u;  /* the watch byte */
        p.tail_len = 1;
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
    return frame_drive(ctx, src, o, multi, g, p.per_rec, 1, slot_bytes, fb, out, [&](const FrameGeom &G) {
        p.out_bytes = G.out_bytes;
        p.out_off = G.out_off;
        p.out_capacity = G.total;
        p.status = G.status;
        p.path_cap = G.path_cap;
        p.json_cap = G.json_cap;
        p.path_limit = G.path_limit;
        p.json_limit = G.json_limit;
        return multi ? (has_data ? launch_jute<true, true>(ctx, p, G.smem) : launch_jute<true, false>(ctx, p, G.smem))
                     : (has_data ? launch_jute<false, true>(ctx, p, G.smem) : launch_jute<false, false>(ctx, p, G.smem));
    });
}

template <bool MULTI, bool DATA, bool PAIR>
static int launch_jute_entry(regk_ctx *ctx, const JuteEntryParams &p, size_t smem)
{
    const int rc = set_smem_limit(ctx, (const void *)regk_jute_entry_kernel<MULTI, DATA, PAIR>, smem);
    if (rc)
        return rc;
    regk_jute_entry_kernel<MULTI, DATA, PAIR><<<(unsigned)((p.n + JUTE_TILE - 1) / JUTE_TILE), JUTE_THREADS, smem, ctx->stream>>>(p);
    CK(cudaGetLastError());
    return REGK_OK;
}

/* Frames whose entries carry a version of their own (`version`: [n] device array, NULL = o->version for all) or that
   pair a delete with a create (`pair`: REGK_ZK_REPLACE, always multi transactions) - regk_jute_entry_kernel.  Output
   and buffers as frame_requests. */
static int frame_entry_requests(regk_ctx *ctx, const FrameSrc &src, const regk_jute_opts *o, const int32_t *version, bool pair,
    FrameBufs &fb, regk_frames *out)
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
    return frame_drive(ctx, src, o, multi, g, p.per_rec, pair ? 2 : 1, JUTE_TILE * JUTE_ESLOT, fb, out, [&](const FrameGeom &G) {
        p.out_bytes = G.out_bytes;
        p.out_off = G.out_off;
        p.out_capacity = G.total;
        p.status = G.status;
        p.path_cap = G.path_cap;
        p.json_cap = G.json_cap;
        p.path_limit = G.path_limit;
        p.json_limit = G.json_limit;
        return pair ? launch_jute_entry<true, true, true>(ctx, p, G.smem)
            : multi ? (has_data ? launch_jute_entry<true, true, false>(ctx, p, G.smem) : launch_jute_entry<true, false, false>(ctx, p, G.smem))
                    : (has_data ? launch_jute_entry<false, true, false>(ctx, p, G.smem) : launch_jute_entry<false, false, false>(ctx, p, G.smem));
    });
}

/* What a successful write framing framed, for regk_read_results: src's entries in `frames` frames of o->group (0 counts
   as 1), its paths and data where src has them, what each entry stands for (`subject`, NULL = itself), and the
   generation of the state src lives in. */
static void record_framing(regk_ctx::ResDesc &d, const FrameSrc &src, const regk_jute_opts *o, uint32_t op, bool multi,
    uint64_t frames, const unsigned long long *subject, uint64_t gen)
{
    d.valid = true;
    d.f = ResFraming{};
    d.f.xid_base = o->xid_base;
    d.f.op = op;
    d.f.group = o->group ? o->group : 1u;
    d.f.multi = multi ? 1u : 0u;
    d.f.frames = frames;
    d.f.entries = src.n;
    d.f.path_bytes = src.path_bytes;
    d.f.path_off = src.path_off;
    d.f.data_off = src.json_off;
    d.subject = subject;
    d.tol = op == REGK_ZK_DELETE ? -101 : 0;    /* NONODE: cleanupPreviousEntries ignores it (lib/register.js:88) */
    d.gen = gen;
}

/* regk_parents.cuh on the path stream of the batch finished last (n >= 1 records), into the given buffers: enqueues
   the table reset, `start` (if any) and the three kernels on the context's stream; p->parent_len / unique_first / n_unique are device
   pointers into `len` and `unique`. */
static int enqueue_parent_pass(regk_ctx *ctx, ParentPass &b, uint64_t n, cudaEvent_t start, ParentParams *out)
{
    cudaStream_t s = ctx->stream;
    DevBuf &len = b.len, &slot = b.slot, &table = b.table, &totals = b.totals, &unique = b.unique;
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
    p.path_bytes = ctx->last.path_bytes;
    p.path_off = ctx->last.path_off;
    p.parent_len = (uint32_t *)len.p;
    p.slot_of = (uint32_t *)slot.p;
    p.owner = (uint32_t *)table.p;
    p.mask = (uint32_t)(slots - 1);
    p.tile_total = (uint32_t *)totals.p;
    p.super_total = (unsigned long long *)((uint8_t *)totals.p + ((ntiles * 4 + 15) & ~(size_t)15));
    p.unique_first = (unsigned long long *)unique.p;
    p.n_unique = p.unique_first + n;
    p.tail_mode = ctx->last.alias ? 0u : (ctx->last.host_off ? 2u : 1u);
    p.host_stride = ctx->last.host_stride;
    p.host_off = ctx->last.host_off;
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
    regk_ctx *const ctx = nullptr;              /* errors before the context exists go to regk_last_error(NULL) */
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
    auto c = std::make_unique<regk_ctx>();
    c->device = device;
    CK(cudaSetDevice(device));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)     /* sm_90a code runs on compute capability 9.0 only */
        return fail(nullptr, REGK_ERR_CUDA, "regk_create: device %d is sm_%d%d; this build targets sm_90a (H100)",
            device, prop.major, prop.minor);
    c->sm_count = prop.multiProcessorCount;
    c->max_smem_optin = (int)prop.sharedMemPerBlockOptin;
    int rc;
    if ((rc = ensure_stream(ctx, c->own_stream)) || (rc = ensure_host(ctx, c->h_status_block, sizeof(DevStatus) * regk_ctx::NSLOTS)))
        return rc;
    c->stream = c->own_stream;
    memset(c->h_status_block.p, 0, sizeof(DevStatus) * regk_ctx::NSLOTS);
    for (int i = 0; i < regk_ctx::NSLOTS; i++) {
        for (Event &ev : c->slots[i].ev)
            if ((rc = ensure_event(ctx, ev)))
                return rc;
        c->slots[i].h_status = (DevStatus *)c->h_status_block.p + i;
    }
    *out = c.release();
    return REGK_OK;
}

void regk_destroy(regk_ctx *ctx)
{
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
                                  "mkdirp_tight_table", "reconcile_tight_table", "stats_cand_shared", nullptr};
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
    if (!strcmp(name, "walk_resolve_segments"))
        return (int64_t)ctx->wr.segments;
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
    uint32_t *flag = (uint32_t *)ctx->h_gather_flag.p;
    if (flag && *flag) {
        *flag = 0;
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
    int rc = ensure_gather_flag(ctx);
    if (rc)
        return rc;
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
    p.flag = (uint32_t *)ctx->h_gather_flag.p;
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
    int rc;
    if ((rc = ensure_dev(ctx, ctx->job_bases, (size_t)regk_ctx::NSLOTS * 64)) ||
        (rc = ensure_host(ctx, ctx->h_job_bases, (size_t)regk_ctx::NSLOTS * 64)) || (rc = ensure_gather_flag(ctx)))
        return rc;
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
    e.host_flag = (uint32_t *)ctx->h_gather_flag.p;
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
    const bool two_deep = !in_dev && !out_dev && async && n;
    regk_ctx::HostSet &hs = two_deep ? ctx->hset[ctx->hseq & 1] : ctx->sync_set;
    int rc;
    if (two_deep) {
        for (const auto &sl : ctx->slots)
            if (sl.in_use && sl.set == &hs)
                return fail(ctx, REGK_ERR_STATE,
                    "regk_register_batch: at most two host batches may be in flight; call regk_finish on the older one");
        if ((rc = ensure_stream(ctx, ctx->s_h2d)) || (rc = ensure_stream(ctx, ctx->s_d2h)) ||
            (rc = ensure_event(ctx, hs.e_in, cudaEventDisableTiming)) || (rc = ensure_event(ctx, hs.e_out, cudaEventDisableTiming)))
            return rc;
    }

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
            rc = pipelined ? ensure_dev(ctx, hs.in[i], sz[i] + 16)         /* run_pipelined copies it chunk by chunk */
                           : stage_in(ctx, hs.in[i], src[i], sz[i], two_deep ? ctx->s_h2d : s);
            if (rc)
                return rc;
            dev[i] = hs.in[i].p;
        }
    }
    if (two_deep) {
        /* this set's staging was last read by the kernels of the batch two submissions back, which has been
           finished (checked above); the kernels below wait for the copies */
        CK(cudaEventRecord(hs.e_in, ctx->s_h2d));
        CK(cudaStreamWaitEvent(s, hs.e_in, 0));
    }

    /* ---- outputs (capacity = exact upper bounds, see DESIGN.md) ---- */
    const uint64_t path_cap = do_path ? dom_len + host_len + 2 * n + 16 : 16;
    const uint64_t json_cap = do_json ? n * (uint64_t)(38 + 2 * ctx->max_type_q + 4 + 18 + 11) + 2 * addr_len +
        11 * ports_len + 16 : 16;
    if (!job && ((rc = ensure_dev(ctx, hs.path_bytes, path_cap)) || (rc = ensure_dev(ctx, hs.path_off, (n + 1) * 8)) ||
        (rc = ensure_dev(ctx, hs.json_bytes, json_cap)) || (rc = ensure_dev(ctx, hs.json_off, (n + 1) * 8))))
        return rc;
    /* job step: the outputs are the rank's own whole-job buffers, every position job-absolute */
    const regk_job &J = ctx->job;
    uint8_t *const out_path_bytes = job ? (uint8_t *)J.path_bytes[J.rank] : (uint8_t *)hs.path_bytes.p;
    unsigned long long *const out_path_off = job ? (unsigned long long *)J.path_off[J.rank] + J.rec_base : (unsigned long long *)hs.path_off.p;
    uint8_t *const out_json_bytes = job ? (uint8_t *)J.json_bytes[J.rank] : (uint8_t *)hs.json_bytes.p;
    unsigned long long *const out_json_off = job ? (unsigned long long *)J.json_off[J.rank] + J.rec_base : (unsigned long long *)hs.json_off.p;
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
        if ((rc = ensure_stream(ctx, ctx->s_side)) || (rc = ensure_event(ctx, ctx->ws_clean[ring], cudaEventDisableTiming)))
            return rc;
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
        CK(cudaMemsetAsync(hs.path_off.p, 0, 8, s));
        CK(cudaMemsetAsync(hs.json_off.p, 0, 8, s));
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
        /* the exact-offset redo (regk_finish) launches the exact variant with the same budget */
        const void *kernel = alias ? (const void *)regk_path_kernel<true, false> : (const void *)regk_path_kernel<false, false>;
        const void *exact = alias ? (const void *)regk_path_kernel<true, true> : (const void *)regk_path_kernel<false, true>;
        if ((rc = set_smem_limit(ctx, kernel, path_smem)) || (rc = set_smem_limit(ctx, exact, path_smem)) ||
            (rc = lookahead_tiles(ctx, alias ? 0 : 1, kernel, path_smem, &pp.lookahead)))
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
        if ((rc = set_smem_limit(ctx, (const void *)regk_json_kernel, json_smem)) ||
            (rc = lookahead_tiles(ctx, 2, (const void *)regk_json_kernel, json_smem, &jp.lookahead)))
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
            hp.dev[i] = need[i] && src[i] ? hs.in[i].p : nullptr;
        }
        slot.set = &hs;
        rc = run_pipelined(ctx, *slot.set, b, res, pp, path_smem, jp, json_smem, hp);
        ctx->skip.last = {};
        if (rc == REGK_ERR_OUT_OF_DOMAIN && (b->flags & REGK_SKIP_BAD) && !(res->bad_bits & REGK_BAD_TOO_LARGE)) {
            /* the whole batch is staged in its set: redo it from there like a dirty batch in regk_finish */
            slot.n = n;
            slot.flags = b->flags;
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
            ctx->skip.last.valid = true;
            ctx->skip.last.n = n;
        }
        if (rc == REGK_OK)
            set_last(ctx, do_path ? pp.out_bytes : nullptr, do_path ? pp.out_off : nullptr, do_json ? jp.out_bytes : nullptr,
                do_json ? jp.out_off : nullptr, n, pp.host_off, pp.host_stride, alias);
        if (rc != REGK_ERR_STATE + 100)         /* anything but "needs the exact redo" */
            return rc;
        /* some domain has empty labels: run the whole batch again through the regular (exact-capable) path */
        for (int i = 0; i < 11; i++)
            if (dev[i] && sz[i])
                CK(cudaMemcpyAsync(hs.in[i].p, src[i], sz[i], cudaMemcpyHostToDevice, s));
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
        if (do_path && (rc = narrow_offsets(ctx, hs.path_off.p, hs.off32_p, n, s)))
            return rc;
        if (do_json && (rc = narrow_offsets(ctx, hs.json_off.p, hs.off32_j, n, s)))
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
            CK(cudaMemcpyAsync((unsigned long long *)ctx->h_job_bases.p + 8 * (ctx->seq % regk_ctx::NSLOTS), d_bases, 64,
                cudaMemcpyDeviceToHost, ctx->s_side));
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

    slot.set = &hs;
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
    if (two_deep) {
        /* the other set's batch, if still open: its kernels ran ahead of this batch's copies - start its D2H now
           so that it overlaps this batch's H2D */
        ctx->hseq++;
        for (auto &sl : ctx->slots)
            if (&sl != &slot && sl.in_use && ctx->is_async(sl.set) && !sl.d2h_issued) {
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
 * Fence pass -> compaction of the kept records into ctx->skip.in -> that batch through regk_register_batch as an
 * ordinary device batch (its outputs, in sync_set.path_bytes / json_bytes, are the result's streams and what the
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
        bool ok = ctx->is_async(slot->set);
        for (const auto &sl : ctx->slots)
            if (sl.in_use && !ctx->is_async(sl.set))
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
    if ((rc = ensure_dev(ctx, ctx->skip.work, bits_off + align16(n) + 16)) || (rc = ensure_host(ctx, ctx->skip.h_status, sizeof(SkipStatus))))
        return rc;
    uint8_t *wk = (uint8_t *)ctx->skip.work.p;
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
    CK(cudaMemcpyAsync(ctx->skip.h_status.p, sp.status, sizeof(SkipStatus), cudaMemcpyDeviceToHost, s));
    cudaError_t e = cudaStreamSynchronize(s);
    if (e != cudaSuccess)
        return fail(ctx, REGK_ERR_CUDA, "skip-mode fence pass failed: %s", cudaGetErrorString(e));
    const SkipStatus fs = *(const SkipStatus *)ctx->skip.h_status.p;
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
        if ((rc = ensure_dev(ctx, ctx->skip.in[i], csz[i] + 16)))
            return rc;
        cin[i] = ctx->skip.in[i].p;
    }
    if ((rc = ensure_dev(ctx, ctx->skip.index, nskip * 8 + 16)) || (rc = ensure_dev(ctx, ctx->skip.bits, nskip + 16)))
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
    sp.skip_index = (unsigned long long *)ctx->skip.index.p;
    sp.skip_bits = (uint8_t *)ctx->skip.bits.p;
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
    if ((rc = ensure_dev(ctx, ctx->skip.off_p, (n + 1) * 8)) || (rc = ensure_dev(ctx, ctx->skip.off_j, (n + 1) * 8)))
        return rc;
    ExpandParams ep{};
    ep.n = n;
    ep.bits = sp.bits;
    ep.tile_total = sp.tile_total[SKIP_REC];
    ep.super_total = sp.super_total[SKIP_REC];
    ep.c_path_off = do_path ? (const unsigned long long *)cres.path_off : nullptr;
    ep.c_json_off = do_json ? (const unsigned long long *)cres.json_off : nullptr;
    ep.path_off = (unsigned long long *)ctx->skip.off_p.p;
    ep.json_off = (unsigned long long *)ctx->skip.off_j.p;
    regk_expand_kernel<<<(unsigned)(n / TILE + 1), TILE, 0, s>>>(ep);
    CK(cudaGetLastError());
    if (!do_path)
        CK(cudaMemsetAsync(ctx->skip.off_p.p, 0, (n + 1) * 8, s));
    if (!do_json)
        CK(cudaMemsetAsync(ctx->skip.off_j.p, 0, (n + 1) * 8, s));
    uint32_t launches = slot->launches + 3 + cres.launches;
    regk_ctx::HostSet &hs = *slot->set;
    const bool off32 = slot->off32 && !out_dev && cres.path_total < (1ull << 32) && cres.json_total < (1ull << 32);
    if (off32) {
        if ((rc = narrow_offsets(ctx, ctx->skip.off_p.p, hs.off32_p, n, s)) || (rc = narrow_offsets(ctx, ctx->skip.off_j.p, hs.off32_j, n, s)))
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
        res->path_off = (uint64_t *)ctx->skip.off_p.p;
        res->json_bytes = cres.json_bytes;
        res->json_off = (uint64_t *)ctx->skip.off_j.p;
        e = cudaStreamSynchronize(s);
        if (e != cudaSuccess)
            return fail(ctx, REGK_ERR_CUDA, "skip-mode offset expansion failed: %s", cudaGetErrorString(e));
    } else {
        if ((rc = ensure_host(ctx, hs.h_path_bytes, cres.path_total + 16)) || (rc = ensure_host(ctx, hs.h_path_off, (n + 1) * 8)) ||
            (rc = ensure_host(ctx, hs.h_json_bytes, cres.json_total + 16)) || (rc = ensure_host(ctx, hs.h_json_off, (n + 1) * 8)))
            return rc;
        const size_t ow = off32 ? 4 : 8;
        if (do_path) {
            CK(cudaMemcpyAsync(hs.h_path_bytes.p, cres.path_bytes, cres.path_total, cudaMemcpyDeviceToHost, s));
            CK(cudaMemcpyAsync(hs.h_path_off.p, off32 ? hs.off32_p.p : ctx->skip.off_p.p, (n + 1) * ow, cudaMemcpyDeviceToHost, s));
        } else {
            memset(hs.h_path_off.p, 0, (n + 1) * 8);
        }
        if (do_json) {
            CK(cudaMemcpyAsync(hs.h_json_bytes.p, cres.json_bytes, cres.json_total, cudaMemcpyDeviceToHost, s));
            CK(cudaMemcpyAsync(hs.h_json_off.p, off32 ? hs.off32_j.p : ctx->skip.off_j.p, (n + 1) * ow, cudaMemcpyDeviceToHost, s));
        } else {
            memset(hs.h_json_off.p, 0, (n + 1) * 8);
        }
        e = cudaStreamSynchronize(s);
        if (e != cudaSuccess)
            return fail(ctx, REGK_ERR_CUDA, "skip-mode result copy failed: %s", cudaGetErrorString(e));
        host_results(res, hs, off32);
    }
    ctx->skip.last.valid = true;
    ctx->skip.last.n = n;
    ctx->skip.last.n_skipped = nskip;
    ctx->skip.last.bad_bits = fs.bad_bits;
    return REGK_OK;
}

int regk_skipped_records(regk_ctx *ctx, uint32_t flags, regk_skipped *out)
{
    if (!ctx || !out)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_skipped_records: NULL argument");
    if (!ctx->skip.last.valid)
        return fail(ctx, REGK_ERR_STATE, "regk_skipped_records: the batch finished last was not a REGK_SKIP_BAD batch");
    memset(out, 0, sizeof *out);
    const regk_ctx::Skip::Last &sl = ctx->skip.last;
    out->n = sl.n;
    out->n_skipped = sl.n_skipped;
    out->bad_bits = sl.bad_bits;
    if (!sl.n_skipped)
        return REGK_OK;
    if (flags & REGK_OUT_DEVICE) {
        out->flags = REGK_OUT_DEVICE;
        out->index = (const uint64_t *)ctx->skip.index.p;
        out->bits = (const uint8_t *)ctx->skip.bits.p;
        return REGK_OK;
    }
    CK(cudaSetDevice(ctx->device));
    int rc;
    if ((rc = to_host(ctx, ctx->skip.h_index, ctx->skip.index.p, sl.n_skipped * 8, ctx->stream)) ||
        (rc = to_host(ctx, ctx->skip.h_bits, ctx->skip.bits.p, sl.n_skipped, ctx->stream)))
        return rc;
    CK(cudaStreamSynchronize(ctx->stream));
    out->index = (const uint64_t *)ctx->skip.h_index.p;
    out->bits = (const uint8_t *)ctx->skip.h_bits.p;
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
        uint32_t *flag = (uint32_t *)ctx->h_gather_flag.p;
        if (flag && *flag == 2u) {
            *flag = 0;
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
        if (ctx->pending && !ctx->is_async(slot->set))      /* device outputs are single-buffered; host sets are not */
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
            const int rc = narrow_offsets(ctx, p.out_off, slot->set->off32_p, p.n, s);
            if (rc)
                return rc;
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
    ctx->skip.last = regk_ctx::Skip::Last{};
    if (slot->flags & REGK_SKIP_BAD) {
        if (st.bad_bits && !(st.bad_bits & REGK_BAD_TOO_LARGE) && !st.overflow)
            return finish_skip(ctx, slot, st, res);
        if (!st.bad_bits) {
            ctx->skip.last.valid = true;
            ctx->skip.last.n = n;
        }
    }
    const bool ok = !st.bad_bits;
    set_last(ctx, ok ? slot->dev_path_bytes : nullptr, ok ? slot->dev_path_off : nullptr, ok ? slot->dev_json_bytes : nullptr,
        ok ? slot->dev_json_off : nullptr, n, slot->dev_host_off, slot->host_stride, slot->alias);
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
        const unsigned long long *hb = (const unsigned long long *)ctx->h_job_bases.p + 8 * ((size_t)(slot - ctx->slots));
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
    regk_ctx::HostSet &hs = *slot->set;
    if (out_dev) {
        res->flags = REGK_OUT_DEVICE;
        res->path_bytes = (uint8_t *)hs.path_bytes.p;
        res->path_off = (uint64_t *)hs.path_off.p;
        res->json_bytes = (uint8_t *)hs.json_bytes.p;
        res->json_off = (uint64_t *)hs.json_off.p;
        return REGK_OK;
    }
    int rc;
    if (ctx->is_async(&hs)) {
        if (!slot->d2h_issued && (rc = issue_d2h(ctx, *slot)))
            return rc;
        e = cudaEventSynchronize(hs.e_out);
        if (e != cudaSuccess)
            return fail(ctx, REGK_ERR_CUDA, "device-to-host copy failed: %s", cudaGetErrorString(e));
    } else {
        if ((rc = enqueue_d2h(ctx, *slot, s)))
            return rc;
        CK(cudaStreamSynchronize(s));
    }
    host_results(res, hs, slot->off32);
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
            if ((rc = stage_in(ctx, ctx->svc.in[i], src[i], sz[i], s)))
                return rc;
            dev[i] = ctx->svc.in[i].p;
        }
    }
    /* 58 fixed + 3 commas + '}}}' + "srvce":"" + "proto":"" + "port": + 10 digits + "ttl": + '-' and 10 digits */
    const uint64_t cap = n * (uint64_t)(58 + 3 + 3 + 10 + 10 + 7 + 10 + 6 + 11) + srvce_len + proto_len + 16;
    const uint64_t ntiles = (n + TILE - 1) / TILE;
    const size_t totals_off = 128, super_off = (totals_off + ntiles * 4 + 15) & ~(size_t)15;
    const size_t work_bytes = super_off + (ntiles / SUPER + 1) * 8 + 64;
    regk_ctx::HostSet &os = ctx->sync_set;      /* the payloads go where a batch's payloads go */
    if ((rc = ensure_dev(ctx, os.json_bytes, cap)) || (rc = ensure_dev(ctx, os.json_off, (n + 1) * 8)) ||
        (rc = ensure_dev(ctx, ctx->svc.work, work_bytes)))
        return rc;
    uint8_t *wk = (uint8_t *)ctx->svc.work.p;
    CK(cudaMemsetAsync(wk, 0, work_bytes, s));
    if (n == 0)
        CK(cudaMemsetAsync(os.json_off.p, 0, 8, s));
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
        p.out_bytes = (uint8_t *)os.json_bytes.p;
        p.out_off = (unsigned long long *)os.json_off.p;
        p.out_capacity = cap;
        p.tile_total = (uint32_t *)(wk + totals_off);
        p.super_total = (unsigned long long *)(wk + super_off);
        p.status = (DevStatus *)wk;
        p.srvce_limit = srvce_len;
        p.proto_limit = proto_len;
        const uint64_t mean = 58 + 3 + 3 + 20 + 13 + 17 + (srvce_len + proto_len) / n + 2;
        p.out_cap = (uint32_t)align16(std::min<uint64_t>(mean * TILE * 9 / 8 + 512, 98304));
        const size_t smem = (size_t)p.out_cap + 32;
        if ((rc = set_smem_limit(ctx, (const void *)regk_service_kernel, smem)))
            return rc;
        CK(cudaEventRecord(slot.ev[0], s));
        regk_service_len_kernel<<<(unsigned)std::min<uint64_t>(ntiles, (uint64_t)ctx->sm_count * 8), TILE, 0, s>>>(p, (uint32_t)ntiles);
        CK(cudaGetLastError());
        regk_service_kernel<<<(unsigned)ntiles, TILE, smem, s>>>(p);
        CK(cudaGetLastError());
        CK(cudaEventRecord(slot.ev[1], s));
        launches = 2;
    }
    CK(cudaMemcpyAsync(slot.h_status, wk, sizeof(DevStatus), cudaMemcpyDeviceToHost, s));
    if ((rc = sync_or_fail(ctx, s, "regk_service_records")))
        return rc;
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
    set_last(ctx, nullptr, nullptr, nullptr, nullptr, 0, nullptr, 0, false);      /* the payload buffers were reused */
    if (out_dev) {
        res->flags = REGK_OUT_DEVICE;
        res->json_bytes = (uint8_t *)os.json_bytes.p;
        res->json_off = (uint64_t *)os.json_off.p;
        return REGK_OK;
    }
    if ((rc = to_host(ctx, os.h_json_bytes, os.json_bytes.p, st.json_total, s)) ||
        (rc = to_host(ctx, os.h_json_off, os.json_off.p, (n + 1) * 8, s)))
        return rc;
    CK(cudaStreamSynchronize(s));
    res->json_bytes = (uint8_t *)os.h_json_bytes.p;
    res->json_off = (uint64_t *)os.h_json_off.p;
    return REGK_OK;
}

/* The watch state of the batch finished last: a new batch generation starts with no kinds, nothing in flight and the
   SetWatches gate closed (the zxid high-water mark stays). */
static regk_ctx::Watch &watch_state(regk_ctx *ctx)
{
    regk_ctx::Watch &w = ctx->wq;
    if (w.gen != ctx->last.gen) {
        w.gen = ctx->last.gen;
        w.rec_n = w.dir_d = 0;
        w.ex_watch = w.ch_watch = w.ex_fly = w.ch_fly = w.gate = w.lmax_ok = false;
    }
    return w;
}

/* the kinds of the generation's `count` records (dirs == false) or directories, all NONE when first asked for */
static int watch_kinds(regk_ctx *ctx, bool dirs, uint64_t count, uint8_t **kind)
{
    regk_ctx::Watch &w = watch_state(ctx);
    DevBuf &b = dirs ? w.dir_kind : w.rec_kind;
    uint64_t &have = dirs ? w.dir_d : w.rec_n;
    if (have != count || !b.p) {
        const int rc = ensure_dev(ctx, b, count + 16);
        if (rc)
            return rc;
        CK(cudaMemsetAsync(b.p, 0, count + 16, ctx->stream));
        have = count;
    }
    *kind = (uint8_t *)b.p;
    return REGK_OK;
}

/* The items of the last watched exists (dirs == false) or getChildren framing, if its replies are unread, are in
   flight: their kinds become NONE (a subset's items, or every kind when the framing's list is gone).  Called before a
   framing overwrites that list, and by regk_setwatches_requests; *launches (if given) counts the launch. */
static int watch_forget_unread(regk_ctx *ctx, bool dirs, uint32_t *launches)
{
    regk_ctx::Watch &w = watch_state(ctx);
    bool &fly = dirs ? w.ch_fly : w.ex_fly;
    const uint64_t have = dirs ? w.dir_d : w.rec_n;
    if (!fly || !have) {
        fly = false;
        return REGK_OK;
    }
    uint8_t *kind = (uint8_t *)(dirs ? w.dir_kind : w.rec_kind).p;
    const regk_ctx::Children &ch = ctx->ch;
    const unsigned long long *items = nullptr;
    uint64_t m = 0;
    if (!dirs && ctx->ex_valid && ctx->ex_gen == ctx->last.gen && ctx->ex_sub) {
        items = ctx->ex_rec;
        m = ctx->ex_n;
    } else if (dirs && ch.framed && ch.gen == ctx->last.gen && ch.sub_item) {
        items = ch.sub_item;
        m = ch.d;
    } else {
        CK(cudaMemsetAsync(kind, 0, have, ctx->stream));
    }
    if (items && m) {
        regk_watch_forget_kernel<<<(unsigned)((m + 255) / 256), 256, 0, ctx->stream>>>(items, m, kind);
        CK(cudaGetLastError());
        if (launches)
            ++*launches;
    }
    fly = false;
    return REGK_OK;
}

/* an exists (dirs == false) or getChildren framing was made, with the watch byte or without */
static int watch_framed(regk_ctx *ctx, bool dirs, bool watched)
{
    const int rc = watch_forget_unread(ctx, dirs, nullptr);
    if (rc)
        return rc;
    regk_ctx::Watch &w = ctx->wq;
    (dirs ? w.ch_watch : w.ex_watch) = watched;
    (dirs ? w.ch_fly : w.ex_fly) = watched;
    return REGK_OK;
}

/* a read of the last exists / getChildren framing succeeded: with the watch byte, reply k (err[k], k < m) gives item
   sub[k] (or k) of the generation's `count` its kind.  The launch is the bookkeeping's, not the read's. */
static int watch_read(regk_ctx *ctx, bool dirs, const int32_t *err, uint64_t m, const unsigned long long *sub, uint64_t count)
{
    regk_ctx::Watch &w = watch_state(ctx);
    if (!(dirs ? w.ch_watch : w.ex_watch))
        return REGK_OK;
    uint8_t *kind = nullptr;
    const int rc = watch_kinds(ctx, dirs, count, &kind);
    if (rc)
        return rc;
    if (m) {
        const WatchKindParams kp{m, err, sub, kind, dirs};
        regk_watch_kind_kernel<<<(unsigned)((m + 255) / 256), 256, 0, ctx->stream>>>(kp);
        CK(cudaGetLastError());
    }
    (dirs ? w.ch_fly : w.ex_fly) = false;
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
    const bool getdata = o->op == REGK_ZK_GETDATA, exists = o->op == REGK_ZK_EXISTS;
    if (o->op != REGK_ZK_CREATE && o->op != REGK_ZK_DELETE && o->op != REGK_ZK_SETDATA && !getdata && !exists)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_jute_requests: op %u is not create (1), delete (2), exists (3), getData (4) "
                                               "or setData (5)", o->op);
    if ((o->flags & REGK_ZK_WATCH) && !getdata && !exists)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_jute_requests: REGK_ZK_WATCH arms a watch with a read; op %u is a write",
            o->op);
    if (o->group > 65536)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_jute_requests: at most 65536 operations per multi transaction");
    if ((getdata || exists) && o->group != 0)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_jute_requests: %s requests cannot go in a multi transaction (group %u)",
            getdata ? "getData" : "exists", o->group);
    const bool has_data = o->op != REGK_ZK_DELETE && !getdata && !exists;
    if (ctx->pending)
        return fail(ctx, REGK_ERR_STATE, "regk_jute_requests: batches are still in flight; finish them first");
    /* an exists frame carries no data, but its replies are classed against the payload lengths (regk_reconcile_stats) */
    const bool need_json = has_data || exists;
    if (!ctx->last.path_off || (need_json && (!ctx->last.json_off || ctx->last.n != ctx->last.json_n)))
        return fail(ctx, REGK_ERR_STATE, "regk_jute_requests: no finished batch with %s on this context",
            need_json ? "both a path and a payload stream" : "a path stream");
    const FrameSrc src{ctx->last.n, ctx->last.path_bytes, ctx->last.path_off, has_data ? ctx->last.json_bytes : nullptr,
                       has_data ? ctx->last.json_off : nullptr};
    int rc = exists ? watch_forget_unread(ctx, false, nullptr) : REGK_OK;
    if (rc)
        return rc;
    rc = frame_requests(ctx, src, o, ctx->frames, out);
    if (rc == REGK_OK && getdata) {
        ctx->gd_valid = true;
        ctx->gd_gen = ctx->last.gen;
        ctx->gd_xid = o->xid_base;
        ctx->gd_n = ctx->last.n;
    } else if (rc == REGK_OK && exists) {
        ctx->ex_valid = true;
        ctx->ex_gen = ctx->last.gen;
        ctx->ex_xid = o->xid_base;
        ctx->ex_n = ctx->last.n;
        ctx->ex_sub = false;
        rc = watch_framed(ctx, false, o->flags & REGK_ZK_WATCH);
    } else if (rc == REGK_OK) {
        record_framing(ctx->rs.batch, src, o, o->op, o->group != 0, out->n, nullptr, ctx->last.gen);
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
        if (!ctx->last.path_off && !ctx->last.json_off)
            return fail(ctx, REGK_ERR_STATE, "regk_decode: no finished batch on this context");
        n = ctx->last.path_off ? ctx->last.n : ctx->last.json_n;
        pb = ctx->last.path_off ? ctx->last.path_bytes : nullptr;
        po = (const uint64_t *)ctx->last.path_off;
        jb = ctx->last.json_off ? ctx->last.json_bytes : nullptr;
        jo = (const uint64_t *)ctx->last.json_off;
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
                if ((rc = stage_in(ctx, ctx->dec.in[i], src[i], sz[i], s)))
                    return rc;
                dev[i] = ctx->dec.in[i].p;
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
    if ((rc = ensure_dev(ctx, ctx->dec.rec, (n + 1) * sizeof(Decoded))) || (rc = ensure_dev(ctx, ctx->dec.dom, path_total + 16)) ||
        (rc = ensure_dev(ctx, ctx->dec.ports, ports_len * 4 + 16)))
        return rc;
    out->n = n;
    out->flags = dev_out ? REGK_OUT_DEVICE : 0;
    out->dom_bytes_len = path_total;
    out->ports_len = ports_len;
    cudaEvent_t e0 = ctx->slots[0].ev[0], e1 = ctx->slots[0].ev[1];
    if (n) {
        DecodeParams p{};
        p.n = n;
        p.path_bytes = po ? (pb ? pb : (const uint8_t *)ctx->dec.dom.p) : nullptr;     /* an empty stream still has offsets */
        p.path_off = (const unsigned long long *)po;
        p.json_bytes = jo ? (jb ? jb : (const uint8_t *)ctx->dec.dom.p) : nullptr;
        p.json_off = (const unsigned long long *)jo;
        p.host_nodes = in->host_nodes;
        p.out = (Decoded *)ctx->dec.rec.p;
        p.dom_bytes = (uint8_t *)ctx->dec.dom.p;
        p.ports = (uint32_t *)ctx->dec.ports.p;
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
        if ((rc = set_smem_limit(ctx, (const void *)regk_decode_kernel, dsmem)))
            return rc;
        CK(cudaEventRecord(e0, s));
        regk_decode_kernel<<<(unsigned)((n + DEC_TILE - 1) / DEC_TILE), DEC_TILE, dsmem, s>>>(p);
        CK(cudaGetLastError());
        CK(cudaEventRecord(e1, s));
        out->launches = 1;
    }
    if ((rc = sync_or_fail(ctx, s, "regk_decode")))
        return rc;
    if (n)
        cudaEventElapsedTime(&out->kernel_ms, e0, e1);
    if (dev_out) {
        out->rec = (const regk_decoded *)ctx->dec.rec.p;
        out->dom_bytes = (const uint8_t *)ctx->dec.dom.p;
        out->ports = (const uint32_t *)ctx->dec.ports.p;
        return REGK_OK;
    }
    if ((rc = ensure_host(ctx, ctx->dec.h_rec, (n + 1) * sizeof(Decoded))) || (rc = ensure_host(ctx, ctx->dec.h_dom, path_total + 16)) ||
        (rc = ensure_host(ctx, ctx->dec.h_ports, ports_len * 4 + 16)))
        return rc;
    if (n) {
        CK(cudaMemcpyAsync(ctx->dec.h_rec.p, ctx->dec.rec.p, n * sizeof(Decoded), cudaMemcpyDeviceToHost, s));
        if (po && path_total)
            CK(cudaMemcpyAsync(ctx->dec.h_dom.p, ctx->dec.dom.p, path_total, cudaMemcpyDeviceToHost, s));
        if (jo)
            CK(cudaMemcpyAsync(ctx->dec.h_ports.p, ctx->dec.ports.p, ports_len * 4, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
    }
    out->rec = (const regk_decoded *)ctx->dec.h_rec.p;
    out->dom_bytes = (const uint8_t *)ctx->dec.h_dom.p;
    out->ports = (const uint32_t *)ctx->dec.h_ports.p;
    return REGK_OK;
}

int regk_parent_dirs(regk_ctx *ctx, uint32_t flags, regk_parents *out)
{
    if (!ctx || !out)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_parent_dirs: NULL argument");
    memset(out, 0, sizeof *out);
    if (ctx->pending)
        return fail(ctx, REGK_ERR_STATE, "regk_parent_dirs: batches are still in flight; finish them first");
    if (!ctx->last.path_off || !ctx->last.path_bytes)
        return fail(ctx, REGK_ERR_STATE, "regk_parent_dirs: no finished batch with a path stream on this context");
    const uint64_t n = ctx->last.n;
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
    if ((rc = ensure_host(ctx, ctx->par.h_count, 8)) || (rc = ensure_event(ctx, ctx->par.ev[0])) || (rc = ensure_event(ctx, ctx->par.ev[1])))
        return rc;
    cudaEvent_t e0 = ctx->par.ev[0], e1 = ctx->par.ev[1];
    ParentParams p{};
    if ((rc = enqueue_parent_pass(ctx, ctx->par.pass, n, e0, &p)))
        return rc;
    CK(cudaEventRecord(e1, s));
    CK(cudaMemcpyAsync(ctx->par.h_count.p, p.n_unique, 8, cudaMemcpyDeviceToHost, s));
    if ((rc = sync_or_fail(ctx, s, "regk_parent_dirs")))
        return rc;
    float ms = 0;
    cudaEventElapsedTime(&ms, e0, e1);
    const uint64_t nu = *(const unsigned long long *)ctx->par.h_count.p;
    out->n_unique = nu;
    out->launches = 3;
    out->kernel_ms = ms;
    if (dev_out) {
        out->parent_len = p.parent_len;
        out->unique_first = (const uint64_t *)p.unique_first;
        return REGK_OK;
    }
    if ((rc = to_host(ctx, ctx->par.h_len, p.parent_len, n * 4, s)) || (rc = to_host(ctx, ctx->par.h_unique, p.unique_first, nu * 8, s)))
        return rc;
    CK(cudaStreamSynchronize(s));
    out->parent_len = (const uint32_t *)ctx->par.h_len.p;
    out->unique_first = (const uint64_t *)ctx->par.h_unique.p;
    return REGK_OK;
}

int regk_mkdirp_dirs(regk_ctx *ctx, uint32_t flags, regk_dirs *out)
{
    if (!ctx || !out)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_mkdirp_dirs: NULL argument");
    memset(out, 0, sizeof *out);
    if (ctx->pending)
        return fail(ctx, REGK_ERR_STATE, "regk_mkdirp_dirs: batches are still in flight; finish them first");
    if (!ctx->last.path_off || !ctx->last.path_bytes)
        return fail(ctx, REGK_ERR_STATE, "regk_mkdirp_dirs: no finished batch with a path stream on this context");
    const uint64_t n = ctx->last.n;
    if (n >= 0xFFFFFFFEull)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_mkdirp_dirs: batch too large");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    const bool dev_out = flags & REGK_OUT_DEVICE;
    ctx->mk.valid = false;
    ctx->mk.gen++;
    regk_ctx::Mkdirp &mk = ctx->mk;
    int rc;
    if ((rc = ensure_host(ctx, mk.h_count, 64)) || (rc = ensure_dev(ctx, mk.count, 64)))
        return rc;
    for (Event &ev : mk.ev)
        if ((rc = ensure_event(ctx, ev)))
            return rc;
    unsigned long long *hc = (unsigned long long *)mk.h_count.p;
    unsigned long long *dc = (unsigned long long *)mk.count.p;
    auto read_counters = [&](const void *src, size_t bytes) -> int {
        CK(cudaMemcpyAsync(hc, src, bytes, cudaMemcpyDeviceToHost, s));
        return sync_or_fail(ctx, s, "regk_mkdirp_dirs");
    };
    std::vector<uint64_t> depth_off(1, 0);
    uint64_t n_invalid = 0, n_dirs = 0, bytes = 0;
    uint32_t launches = 0;
    float ms[3] = {0, 0, 0};
    if (n) {
        /* 1. the distinct immediate directories, on buffers of its own (regk_parent_dirs' results stay as they are) */
        ParentParams pp{};
        if ((rc = enqueue_parent_pass(ctx, mk.pass, n, mk.ev[0], &pp)))
            return rc;
        launches += 3;
        CK(cudaEventRecord(mk.ev[1], s));
        if ((rc = read_counters(pp.n_unique, 8)))
            return rc;
        const uint64_t nu = hc[0];
        /* workspace for up to nu items per pass: flags, two work lists, two-level totals of two counts */
        const uint64_t ntiles = (nu + MK_TILE - 1) / MK_TILE, tt = align16(ntiles * 4), st = (ntiles / SUPER + 1) * 8;
        const size_t totals_bytes = 2 * tt + 2 * st + 16;
        if ((rc = ensure_dev(ctx, mk.flags, nu + 16)) || (rc = ensure_dev(ctx, mk.list[0], nu * 16 + 16)) ||
            (rc = ensure_dev(ctx, mk.list[1], nu * 16 + 16)) || (rc = ensure_dev(ctx, mk.totals, totals_bytes)) ||
            (rc = ensure_dev(ctx, mk.invalid, nu * 8 + 8)))
            return rc;
        uint8_t *tb = (uint8_t *)mk.totals.p;
        MkdirpParams p{};
        p.path_bytes = ctx->last.path_bytes;
        p.path_off = ctx->last.path_off;
        p.parent_len = pp.parent_len;
        p.unique_first = pp.unique_first;
        p.n_unique = nu;
        p.flags = (uint8_t *)mk.flags.p;
        p.tile_a = (uint32_t *)tb;
        p.tile_b = (uint32_t *)(tb + tt);
        p.super_a = (unsigned long long *)(tb + 2 * tt);
        p.super_b = (unsigned long long *)(tb + 2 * tt + st);
        p.counters = dc;
        p.invalid = (unsigned long long *)mk.invalid.p;
        uint4 *list[2] = {(uint4 *)mk.list[0].p, (uint4 *)mk.list[1].p};
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
        if ((rc = ensure_dev(ctx, mk.table, slots * 8)) || (rc = ensure_dev(ctx, mk.drec, entries * 8 + 8)) ||
            (rc = ensure_dev(ctx, mk.dlen, entries * 4 + 8)))
            return rc;
        p.table = (unsigned long long *)mk.table.p;
        p.mask = (uint32_t)(slots - 1);
        p.dir_rec = (unsigned long long *)mk.drec.p;
        p.dir_len = (uint32_t *)mk.dlen.p;
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
        CK(cudaEventRecord(mk.ev[2], s));
        /* 5. dir_off and the packed bytes */
        const uint64_t dt = (n_dirs + MK_TILE - 1) / MK_TILE, dtt = dt * 8, dst = (dt / SUPER + 1) * 8;
        if ((rc = ensure_dev(ctx, mk.dbytes, bytes + 16)) || (rc = ensure_dev(ctx, mk.doff, (n_dirs + 1) * 8)) ||
            (rc = ensure_dev(ctx, mk.totals, dtt + dst + 16)))
            return rc;
        if (n_dirs) {
            MkGatherParams g{};
            g.n_dirs = n_dirs;
            g.path_bytes = ctx->last.path_bytes;
            g.path_off = ctx->last.path_off;
            g.dir_rec = p.dir_rec;
            g.dir_len = p.dir_len;
            g.tile_total = (unsigned long long *)mk.totals.p;
            g.super_total = (unsigned long long *)((uint8_t *)mk.totals.p + dtt);
            g.dir_bytes = (uint8_t *)mk.dbytes.p;
            g.dir_off = (unsigned long long *)mk.doff.p;
            CK(cudaMemsetAsync(g.super_total, 0, dst, s));
            regk_mkdirp_len_kernel<<<(unsigned)dt, MK_TILE, 0, s>>>(g);
            regk_mkdirp_gather_kernel<<<(unsigned)dt, MK_TILE, 0, s>>>(g);
            CK(cudaGetLastError());
            launches += 2;
        } else {
            CK(cudaMemsetAsync(mk.doff.p, 0, 8, s));
        }
        CK(cudaEventRecord(mk.ev[3], s));
        if ((rc = sync_or_fail(ctx, s, "regk_mkdirp_dirs")))
            return rc;
        for (int k = 0; k < 3; k++)
            cudaEventElapsedTime(&ms[k], mk.ev[k], mk.ev[k + 1]);
    } else {
        if ((rc = ensure_dev(ctx, mk.doff, 8)) || (rc = ensure_dev(ctx, mk.dbytes, 16)) ||
            (rc = ensure_dev(ctx, mk.drec, 8)) || (rc = ensure_dev(ctx, mk.dlen, 8)) ||
            (rc = ensure_dev(ctx, mk.invalid, 8)))
            return rc;
        CK(cudaMemsetAsync(mk.doff.p, 0, 8, s));
    }
    /* depth_off was counted on the host; the device result gets a copy */
    const size_t nd1 = depth_off.size();
    if ((rc = ensure_host(ctx, mk.h_depth, nd1 * 8)) || (rc = ensure_dev(ctx, mk.depth, nd1 * 8)))
        return rc;
    memcpy(mk.h_depth.p, depth_off.data(), nd1 * 8);
    CK(cudaMemcpyAsync(mk.depth.p, mk.h_depth.p, nd1 * 8, cudaMemcpyHostToDevice, s));
    CK(cudaStreamSynchronize(s));
    mk.valid = true;
    mk.n_dirs = n_dirs;
    mk.bytes = bytes;
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
    const void *dsrc[6] = {mk.drec.p, mk.dlen.p, mk.depth.p, mk.dbytes.p, mk.doff.p, mk.invalid.p};
    if (!dev_out) {
        HostBuf *hb[6] = {&mk.h_drec, &mk.h_dlen, &mk.h_depth, &mk.h_dbytes, &mk.h_doff, &mk.h_invalid};
        const size_t sz[6] = {n_dirs * 8, n_dirs * 4, 0, bytes, (n_dirs + 1) * 8, n_invalid * 8};
        for (int k = 0; k < 6; k++) {
            if (k != 2 && (rc = to_host(ctx, *hb[k], dsrc[k], sz[k], s)))       /* depth_off is on the host already */
                return rc;
            dsrc[k] = hb[k]->p;
        }
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
    if (!ctx->mk.valid)
        return fail(ctx, REGK_ERR_STATE, "regk_mkdirp_requests: no directory set on this context; call regk_mkdirp_dirs first");
    CK(cudaSetDevice(ctx->device));
    const uint64_t nd = ctx->mk.n_dirs;
    int rc;
    /* CreateRequest with an empty data buffer: the payload offsets are all zero */
    if ((rc = ensure_dev(ctx, ctx->mk.zero, (nd + 1) * 8)))
        return rc;
    CK(cudaMemsetAsync(ctx->mk.zero.p, 0, (nd + 1) * 8, ctx->stream));
    regk_jute_opts o{};
    o.op = REGK_ZK_CREATE;
    o.flags = flags;
    o.xid_base = xid_base;
    o.zk_flags = zk_flags;
    FrameSrc src{nd, (const uint8_t *)ctx->mk.dbytes.p, (const unsigned long long *)ctx->mk.doff.p,
                 (const uint8_t *)ctx->mk.dbytes.p, (const unsigned long long *)ctx->mk.zero.p};
    src.who = "regk_mkdirp_requests";
    if ((rc = frame_requests(ctx, src, &o, ctx->mk.frames, out)))
        return rc;
    record_framing(ctx->rs.mkdirp, src, &o, REGK_ZK_CREATE, false, out->n, nullptr, ctx->mk.gen);
    ctx->rs.mkdirp.tol = -110;                  /* NODEEXISTS: zkplus' mkdirp tolerates it */
    return REGK_OK;
}

/* What every reconcile's passes share, from the batch finished last (n records), the node count m and whether versions
   are carried: sizes and zeroes the tables, totals, counters and lists and fills *pp but for the observed side (o_*,
   validate, want), which the caller sets first; records the start event. */
static int reconcile_prepare(regk_ctx *ctx, uint64_t n, uint64_t m, bool owned, ReconcileParams *pp)
{
    cudaStream_t s = ctx->stream;
    regk_ctx::Reconcile &rb = ctx->rc;
    ReconcileParams &p = *pp;
    int rc;
    /* the batch's totals */
    unsigned long long tot[2] = {0, 0};
    CK(cudaMemcpyAsync(&tot[0], ctx->last.path_off + n, 8, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(&tot[1], ctx->last.json_off + n, 8, cudaMemcpyDeviceToHost, s));
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
    if ((rc = ensure_dev(ctx, rb.t_obs, so * 4)) || (rc = ensure_dev(ctx, rb.t_des, sd * 4)) ||
        (rc = ensure_dev(ctx, rb.slot_obs, m * 4 + 16)) || (rc = ensure_dev(ctx, rb.hash_obs, m * 4 + 16)) ||
        (rc = ensure_dev(ctx, rb.slot_des, n * 4)) || (rc = ensure_dev(ctx, rb.cls, n + 16)) ||
        (rc = ensure_dev(ctx, rb.match, n * 8)) || (rc = ensure_dev(ctx, rb.obs_cls, m + 16)) ||
        (rc = ensure_dev(ctx, rb.totals, totals_bytes)) || (rc = ensure_dev(ctx, rb.count, counters_bytes)) ||
        (rc = ensure_host(ctx, rb.h_count, counters_bytes)))
        return rc;
    for (int l = 0; l < RC_NLISTS; l++)
        if ((rc = ensure_dev(ctx, rb.list[l], (l == RC_LDELETE ? m : n) * 8 + 8)))
            return rc;
    for (int k = 0; k < RC_NGATHERS; k++)
        if ((rc = ensure_dev(ctx, rb.len[k], (k == RC_GDELETE ? m : n) * 4 + 8)))
            return rc;
    for (int k = 0; owned && k < RC_NVER; k++)
        if ((rc = ensure_dev(ctx, rb.ver[k], (k == RC_VDELETE ? m : n) * 4 + 8)))
            return rc;
    for (Event &ev : rb.ev)
        if ((rc = ensure_event(ctx, ev)))
            return rc;
    p.n = n;
    p.m = m;
    p.d_path = ctx->last.path_bytes;
    p.d_path_off = ctx->last.path_off;
    p.d_json = ctx->last.json_bytes;
    p.d_json_off = ctx->last.json_off;
    p.d_path_limit = tot[0] + 16;                   /* every stream buffer of this library has >= 16 bytes of slack */
    p.d_json_limit = tot[1] + 16;
    for (int k = 0; owned && k < RC_NVER; k++)
        p.ver[k] = (int32_t *)rb.ver[k].p;
    p.mask_o = (uint32_t)(so - 1);
    p.mask_d = (uint32_t)(sd - 1);
    p.t_obs = (uint32_t *)rb.t_obs.p;
    p.t_des = (uint32_t *)rb.t_des.p;
    p.slot_obs = (uint32_t *)rb.slot_obs.p;
    p.hash_obs = (uint32_t *)rb.hash_obs.p;
    p.slot_des = (uint32_t *)rb.slot_des.p;
    p.cls = (uint8_t *)rb.cls.p;
    p.match = (unsigned long long *)rb.match.p;
    p.obs_cls = (uint8_t *)rb.obs_cls.p;
    uint8_t *tb = (uint8_t *)rb.totals.p;
    for (int l = 0; l < RC_NLISTS; l++) {
        const bool del = l == RC_LDELETE;
        p.tile_total[l] = (uint32_t *)(tb + (size_t)l * (ttr + str));
        p.super_total[l] = (unsigned long long *)(tb + (size_t)l * (ttr + str) + (del ? tto : ttr));
        p.list[l] = (unsigned long long *)rb.list[l].p;
    }
    for (int k = 0; k < RC_NGATHERS; k++)
        p.len[k] = (uint32_t *)rb.len[k].p;
    p.counters = (unsigned long long *)rb.count.p;
    p.tiles_r = (uint32_t)tiles_r;
    CK(cudaMemsetAsync(p.t_obs, 0, so * 4, s));
    CK(cudaMemsetAsync(p.t_des, 0, sd * 4, s));
    CK(cudaMemsetAsync(tb, 0, totals_bytes, s));
    CK(cudaMemsetAsync(p.counters, 0, counters_bytes, s));
    CK(cudaMemsetAsync(p.counters, 0xFF, 16, s));   /* no bad node, no duplicate node */
    CK(cudaEventRecord(rb.ev[0], s));
    return REGK_OK;
}

/* What follows a reconcile's compact pass, given its counters on the host (hc): the request sets gathered into the
   library's own streams, the stop event, the outputs on the side `flags` asks for, the context's record of the result. */
static int reconcile_finish(regk_ctx *ctx, const ReconcileParams &p, const unsigned long long *hc, bool owned, uint32_t zk_flags,
    uint32_t flags, uint32_t launches, regk_delta *out, const uint64_t **rep, uint64_t *n_rep, const char *who)
{
    cudaStream_t s = ctx->stream;
    regk_ctx::Reconcile &rb = ctx->rc;
    const uint64_t n = p.n, m = p.m;
    const bool dev_out = flags & REGK_OUT_DEVICE;
    int rc;
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
    if ((rc = ensure_dev(ctx, rb.gtotals, gt * 8 + (gt / SUPER + 1) * 8 + 16)))
        return rc;
    for (int g = 0; g < RC_NGATHERS; g++) {
        const uint64_t c = cnt[g_list[g]], bytes = hc[RC_C_BYTES + g];
        DevBuf &gb = rb.gather[g].bytes, &go = rb.gather[g].off;
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
        gp.tile_total = (unsigned long long *)rb.gtotals.p;
        gp.super_total = gp.tile_total + dt;
        gp.dir_bytes = (uint8_t *)gb.p;
        gp.dir_off = (unsigned long long *)go.p;
        CK(cudaMemsetAsync(gp.super_total, 0, (dt / SUPER + 1) * 8, s));
        regk_mkdirp_len_kernel<<<(unsigned)dt, MK_TILE, 0, s>>>(gp);
        regk_mkdirp_gather_kernel<<<(unsigned)dt, MK_TILE, 0, s>>>(gp);
        CK(cudaGetLastError());
        launches += 2;
    }
    CK(cudaEventRecord(rb.ev[1], s));
    if ((rc = sync_or_fail(ctx, s, who)))
        return rc;
    float ms = 0;
    cudaEventElapsedTime(&ms, rb.ev[0], rb.ev[1]);
    const int NOUT = 3 + RC_NLISTS;                 /* cls, match, obs_cls, then the lists */
    const void *dsrc[NOUT] = {p.cls, p.match, p.obs_cls};
    for (int l = 0; l < RC_NLISTS; l++)
        dsrc[3 + l] = p.list[l];
    if (!dev_out) {
        HostBuf *hb[NOUT] = {&rb.h_cls, &rb.h_match, &rb.h_obs_cls};
        size_t sz[NOUT] = {n, n * 8, m};
        for (int l = 0; l < RC_NLISTS; l++) {
            hb[3 + l] = &rb.h_list[l];
            sz[3 + l] = cnt[l] * 8;
        }
        for (int k = 0; k < NOUT; k++) {
            if ((rc = to_host(ctx, *hb[k], dsrc[k], sz[k], s)))
                return rc;
            dsrc[k] = hb[k]->p;
        }
        CK(cudaStreamSynchronize(s));
    }
    rb.valid = true;
    rb.owned = owned;
    rb.zk_flags = zk_flags;
    for (int l = 0; l < RC_NLISTS; l++)
        rb.n_list[l] = cnt[l];
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

/* regk_reconcile (st == NULL) and regk_reconcile_owned: one implementation, the same four passes; `rep` / `n_rep` receive
   the replace list of the owned call */
static int reconcile_run(regk_ctx *ctx, const regk_decode_in *in, const regk_node_stat *st, uint32_t flags, regk_delta *out,
    const uint64_t **rep, uint64_t *n_rep, const char *who)
{
    ctx->rc.valid = false;
    ctx->rc.gen++;
    if (in->flags & REGK_DECODE_LAST)
        return fail(ctx, REGK_ERR_INVALID_ARG, "%s: REGK_DECODE_LAST names no snapshot; pass the snapshot's streams", who);
    if (ctx->pending)
        return fail(ctx, REGK_ERR_STATE, "%s: batches are still in flight; finish them first", who);
    if (!ctx->last.path_off || !ctx->last.json_off || ctx->last.n != ctx->last.json_n)
        return fail(ctx, REGK_ERR_STATE, "%s: no finished batch with both a path and a payload stream on this context "
                                         "(an empty batch or a REGK_JOB_STEP result leaves none)", who);
    const uint64_t n = ctx->last.n, m = in->n;
    if (n >= 0xFFFFFFFFull || m >= 0xFFFFFFFFull)
        return fail(ctx, REGK_ERR_INVALID_ARG, "%s: %llu records and %llu nodes: both must be below 2^32 - 1", who,
            (unsigned long long)n, (unsigned long long)m);
    const bool in_dev = in->flags & REGK_IN_DEVICE;
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
    regk_ctx::Reconcile &rb = ctx->rc;
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
        for (int k = 0; k < (st ? 6 : 4); k++)
            if ((rc = stage_in(ctx, rb.in[k], src[k], sz[k], s)))
                return rc;
        pb = (const uint8_t *)rb.in[0].p;
        po = (const uint64_t *)rb.in[1].p;
        jb = (const uint8_t *)rb.in[2].p;
        jo = (const uint64_t *)rb.in[3].p;
        if (st) {
            sver = (const int32_t *)rb.in[4].p;
            sown = (const int64_t *)rb.in[5].p;
        }
    } else if (m) {
        if ((path_total && !pb) || (json_total && !jb))
            return fail(ctx, REGK_ERR_INVALID_ARG, "%s: snapshot offsets without bytes", who);
        if (((uintptr_t)pb & 3u) || ((uintptr_t)jb & 3u) || ((uintptr_t)po & 7u) || ((uintptr_t)jo & 7u))
            return fail(ctx, REGK_ERR_INVALID_ARG, "%s: misaligned device snapshot (bytes need 4-byte, offsets 8-byte alignment)", who);
    }
    /* an empty stream is never read; its kernels still get a valid pointer */
    if ((rc = ensure_dev(ctx, rb.in[0], 16)) || (rc = ensure_dev(ctx, rb.in[2], 16)))
        return rc;
    if (!pb)
        pb = (const uint8_t *)rb.in[0].p;
    if (!jb)
        jb = (const uint8_t *)rb.in[2].p;
    ReconcileParams p{};
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
    }
    if ((rc = reconcile_prepare(ctx, n, m, st != nullptr, &p)))
        return rc;
    const uint64_t tiles_r = p.tiles_r, tiles_o = (m + RC_TILE - 1) / RC_TILE;
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
    unsigned long long *hc = (unsigned long long *)rb.h_count.p;
    CK(cudaMemcpyAsync(hc, p.counters, RC_NCOUNTERS * 8, cudaMemcpyDeviceToHost, s));
    if ((rc = sync_or_fail(ctx, s, who)))
        return rc;
    if (hc[RC_C_BAD] != ~0ull)
        return fail(ctx, REGK_ERR_INVALID_ARG, "%s: snapshot offsets are not monotone or reach past the totals at node %llu", who,
            hc[RC_C_BAD]);
    if (hc[RC_C_DUPNODE] != ~0ull)
        return fail(ctx, REGK_ERR_INVALID_ARG, "%s: snapshot node %llu has the path of an earlier node; a registry cannot "
                                               "hold two nodes with one path", who, hc[RC_C_DUPNODE]);
    return reconcile_finish(ctx, p, hc, st != nullptr, st ? st->zk_flags : 0u, flags, launches, out, rep, n_rep, who);
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
    ctx->rc.valid = false;
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
    if (o->flags & REGK_ZK_WATCH)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_reconcile_requests: REGK_ZK_WATCH arms a watch with a read; op %u is a "
                                               "write", o->op);
    if (o->group > 65536)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_reconcile_requests: at most 65536 operations per multi transaction");
    if (replace && o->group > 32768)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_reconcile_requests: at most 32768 replace entries (65536 operations) per "
                                               "multi transaction");
    if (ctx->pending)
        return fail(ctx, REGK_ERR_STATE, "regk_reconcile_requests: batches are still in flight; finish them first");
    if (!ctx->rc.valid)
        return fail(ctx, REGK_ERR_STATE, "regk_reconcile_requests: no reconcile result on this context; call regk_reconcile first");
    if ((replace || observed) && !ctx->rc.owned)
        return fail(ctx, REGK_ERR_STATE, "regk_reconcile_requests: replace frames and observed versions need node stats; the last "
                                         "reconcile was regk_reconcile, call regk_reconcile_owned");
    if (ctx->rc.owned && (replace || o->op == REGK_ZK_CREATE) && o->zk_flags != ctx->rc.zk_flags)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_reconcile_requests: zk_flags %u differs from the CreateMode %u regk_reconcile_owned "
                                               "classified with; nodes created so would be classed REPLACE again", o->zk_flags,
                    ctx->rc.zk_flags);
    CK(cudaSetDevice(ctx->device));
    /* gathered streams: create paths / payloads, update paths / payloads, delete paths, replace paths / payloads */
    const int g = o->op == REGK_ZK_CREATE ? RC_GCREATE : o->op == REGK_ZK_SETDATA ? RC_GUPDATE : replace ? RC_GREPLACE : RC_GDELETE;
    const int l = o->op == REGK_ZK_CREATE ? RC_LCREATE : o->op == REGK_ZK_SETDATA ? RC_LUPDATE : replace ? RC_LREPLACE : RC_LDELETE;
    const uint64_t c = ctx->rc.n_list[l];
    regk_ctx::Reconcile &rb = ctx->rc;
    const bool data = g != RC_GDELETE;
    FrameSrc src{c, (const uint8_t *)rb.gather[g].bytes.p, (const unsigned long long *)rb.gather[g].off.p,
                 data ? (const uint8_t *)rb.gather[g + 1].bytes.p : nullptr,
                 data ? (const unsigned long long *)rb.gather[g + 1].off.p : nullptr};
    src.who = "regk_reconcile_requests";
    int rc;
    if (!replace && !observed) {
        rc = frame_requests(ctx, src, o, rb.frames, out);
    } else {
        const int v = l == RC_LUPDATE ? RC_VUPDATE : l == RC_LREPLACE ? RC_VREPLACE : RC_VDELETE;
        const int32_t *ver = observed ? (const int32_t *)rb.ver[v].p : nullptr;
        rc = frame_entry_requests(ctx, src, o, ver, replace, rb.frames, out);
    }
    if (rc == REGK_OK) {
        const int q = o->op == REGK_ZK_CREATE ? 0 : o->op == REGK_ZK_DELETE ? 1 : o->op == REGK_ZK_SETDATA ? 2 : 3;
        record_framing(ctx->rs.rec[q], src, o, replace ? RS_REPLACE : o->op, replace || o->group != 0, out->n,
            (const unsigned long long *)rb.list[l].p, rb.gen);
    }
    return rc;
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
    if (ctx->gd_gen != ctx->last.gen || !ctx->last.path_off)
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
    regk_ctx::Replies &rb = ctx->rq;
    int rc;
    for (Event &ev : rb.ev)
        if ((rc = ensure_event(ctx, ev)))
            return rc;
    const uint8_t *ds = bytes;
    if (!in_dev) {
        if ((rc = stage_in(ctx, rb.stream, bytes, len, s)))
            return rc;
        ds = (const uint8_t *)rb.stream.p;
    }
    const uint64_t nblk = (len + 15) / 16, tiles_s = (nblk + RP_TILE - 1) / RP_TILE, tiles_r = (n + RP_TILE - 1) / RP_TILE;
    uint64_t slots = 1024;
    while (slots < 2 * n)
        slots <<= 1;
    /* two-level totals of the candidate pass (the chain and node passes get theirs once the candidates are counted) */
    const size_t totals_bytes = align16(tiles_s * 4) + (tiles_s / SUPER + 1) * 8;
    const size_t n8 = n * 8 + 16, n4 = n * 4 + 16;
    if ((rc = ensure_dev(ctx, rb.word, nblk * 4 + 16)) || (rc = ensure_dev(ctx, rb.totals, totals_bytes)) ||
        (rc = ensure_dev(ctx, rb.tile_base, tiles_s * 8 + 16)) || (rc = ensure_dev(ctx, rb.err, n4)) ||
        (rc = ensure_dev(ctx, rb.data_pos, n8)) || (rc = ensure_dev(ctx, rb.dlen, n4)) ||
        (rc = ensure_dev(ctx, rb.ver, n4)) || (rc = ensure_dev(ctx, rb.own, n8)) ||
        (rc = ensure_dev(ctx, rb.slot, n4)) || (rc = ensure_dev(ctx, rb.table, slots * 4)) ||
        (rc = ensure_dev(ctx, rb.count, RQ_NCOUNTERS * 8)) || (rc = ensure_host(ctx, rb.h_count, RQ_NCOUNTERS * 8)))
        return rc;
    RepParams p{};
    p.s = ds;
    p.len = len;
    p.xid_base = xb;
    p.n = n;
    p.word = (uint32_t *)rb.word.p;
    p.tile_total = (uint32_t *)rb.totals.p;
    p.super_total = (unsigned long long *)((uint8_t *)rb.totals.p + align16(tiles_s * 4));
    p.tile_base = (unsigned long long *)rb.tile_base.p;
    p.err = (int32_t *)rb.err.p;
    p.data_pos = (unsigned long long *)rb.data_pos.p;
    p.dlen = (uint32_t *)rb.dlen.p;
    p.ver = (int32_t *)rb.ver.p;
    p.own = (long long *)rb.own.p;
    p.slot = (uint32_t *)rb.slot.p;
    p.d_path = ctx->last.path_bytes;
    p.d_path_off = ctx->last.path_off;
    p.table = (uint32_t *)rb.table.p;
    p.mask_t = (uint32_t)(slots - 1);
    p.counters = (unsigned long long *)rb.count.p;
    unsigned long long *hc = (unsigned long long *)rb.h_count.p;
    CK(cudaMemsetAsync(p.counters, 0, RQ_NCOUNTERS * 8, s));
    CK(cudaMemsetAsync(p.counters + RQ_ERR, 0xFF, 8, s));
    CK(cudaMemsetAsync(p.tile_total, 0, totals_bytes, s));
    CK(cudaEventRecord(rb.ev[0], s));
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
    if ((rc = sync_or_fail(ctx, s, "regk_read_replies")))
        return rc;
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
    if ((rc = ensure_dev(ctx, rb.cand, C * 8 + 16)) || (rc = ensure_dev(ctx, rb.mark, C + 16)) ||
        (rc = ensure_dev(ctx, rb.jump, (size_t)(K + 1) * C * 4 + 16)) ||
        (rc = ensure_dev(ctx, rb.totals2, totals2_bytes)))
        return rc;
    p.cand = (unsigned long long *)rb.cand.p;
    p.marked = (uint8_t *)rb.mark.p;
    p.C = C;
    uint32_t *J = (uint32_t *)rb.jump.p;
    RepParams p2 = p;                                   /* the chain and node passes' totals */
    p2.tile_total = (uint32_t *)rb.totals2.p;
    p2.super_total = (unsigned long long *)((uint8_t *)rb.totals2.p + align16(tiles2 * 4));
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
    if ((rc = sync_or_fail(ctx, s, "regk_read_replies")))
        return rc;
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
    if ((rc = ensure_dev(ctx, rb.node_rec, n8)) || (rc = ensure_dev(ctx, rb.node_ver, n4)) ||
        (rc = ensure_dev(ctx, rb.node_own, n8)) || (rc = ensure_dev(ctx, rb.node_plen, n4)) ||
        (rc = ensure_dev(ctx, rb.node_dlen, n4)))
        return rc;
    p.node_rec = (unsigned long long *)rb.node_rec.p;
    p.node_ver = (int32_t *)rb.node_ver.p;
    p.node_own = (long long *)rb.node_own.p;
    p.node_plen = (uint32_t *)rb.node_plen.p;
    p.node_dlen = (uint32_t *)rb.node_dlen.p;
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
    if ((rc = sync_or_fail(ctx, s, "regk_read_replies")))
        return rc;
    const uint64_t m = hc[RQ_M];
    /* 5. the snapshot's streams: node paths from the batch, node data from the reply stream */
    const uint64_t gt = (m + MK_TILE - 1) / MK_TILE;
    if ((rc = ensure_dev(ctx, rb.gtotals, gt * 8 + (gt / SUPER + 1) * 8 + 16)) ||
        (rc = ensure_dev(ctx, rb.snap_off[0], (m + 1) * 8)) || (rc = ensure_dev(ctx, rb.snap_off[1], (m + 1) * 8)))
        return rc;
    uint64_t totals[2] = {0, 0};
    for (int g = 0; g < 2; g++) {
        DevBuf &gb = rb.snap_bytes[g], &go = rb.snap_off[g];
        MkGatherParams gp{};
        gp.n_dirs = m;
        gp.path_bytes = g ? ds : ctx->last.path_bytes;
        gp.path_off = g ? p.data_pos : ctx->last.path_off;
        gp.dir_rec = p.node_rec;
        gp.dir_len = g ? p.node_dlen : p.node_plen;
        gp.tile_total = (unsigned long long *)rb.gtotals.p;
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
    CK(cudaEventRecord(rb.ev[1], s));
    if ((rc = sync_or_fail(ctx, s, "regk_read_replies")))
        return rc;
    float ms = 0;
    cudaEventElapsedTime(&ms, rb.ev[0], rb.ev[1]);
    const int32_t *err_out = p.err;
    const uint64_t *rec_out = (const uint64_t *)p.node_rec;
    if (!dev_out) {
        if ((rc = to_host(ctx, rb.h_err, p.err, n * 4, s)) || (rc = to_host(ctx, rb.h_node, p.node_rec, m * 8, s)))
            return rc;
        CK(cudaStreamSynchronize(s));
        err_out = (const int32_t *)rb.h_err.p;
        rec_out = (const uint64_t *)rb.h_node.p;
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
    out->snapshot.path_bytes = (const uint8_t *)rb.snap_bytes[0].p;
    out->snapshot.path_off = (const uint64_t *)rb.snap_off[0].p;
    out->snapshot.json_bytes = (const uint8_t *)rb.snap_bytes[1].p;
    out->snapshot.json_off = (const uint64_t *)rb.snap_off[1].p;
    out->version = p.node_ver;
    out->ephemeral_owner = (const int64_t *)p.node_own;
    out->kernel_ms = ms;
    return REGK_OK;
}

/* The strings (path_bytes at path_off[rec[k]], len[k] bytes), k < m, packed into `bytes` / `off` by the mkdirp gather pair
   (regk_mkdirp.cuh); *total = their byte count.  Synchronises once to size `bytes`. */
static int pack_strings(regk_ctx *ctx, uint64_t m, const uint8_t *path_bytes, const unsigned long long *path_off,
    const unsigned long long *rec, const uint32_t *len, DevBuf &totals, DevBuf &bytes, DevBuf &off, uint64_t *total,
    uint32_t *launches)
{
    cudaStream_t s = ctx->stream;
    const uint64_t gt = (m + MK_TILE - 1) / MK_TILE;
    int rc;
    *total = 0;
    if ((rc = ensure_dev(ctx, totals, gt * 8 + (gt / SUPER + 1) * 8 + 16)) || (rc = ensure_dev(ctx, off, (m + 1) * 8)))
        return rc;
    if (!m) {
        if ((rc = ensure_dev(ctx, bytes, 16)))
            return rc;
        CK(cudaMemsetAsync(off.p, 0, 8, s));
        return REGK_OK;
    }
    MkGatherParams gp{};
    gp.n_dirs = m;
    gp.path_bytes = path_bytes;
    gp.path_off = path_off;
    gp.dir_rec = rec;
    gp.dir_len = len;
    gp.tile_total = (unsigned long long *)totals.p;
    gp.super_total = gp.tile_total + gt;
    gp.dir_off = (unsigned long long *)off.p;
    CK(cudaMemsetAsync(gp.super_total, 0, (gt / SUPER + 1) * 8, s));
    regk_mkdirp_len_kernel<<<(unsigned)gt, MK_TILE, 0, s>>>(gp);
    std::vector<unsigned long long> gs(gt / SUPER + 1);
    CK(cudaMemcpyAsync(gs.data(), gp.super_total, gs.size() * 8, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    for (unsigned long long v : gs)
        *total += v;
    if ((rc = ensure_dev(ctx, bytes, *total + 16)))
        return rc;
    gp.dir_bytes = (uint8_t *)bytes.p;
    regk_mkdirp_gather_kernel<<<(unsigned)gt, MK_TILE, 0, s>>>(gp);
    CK(cudaGetLastError());
    *launches += 2;
    return REGK_OK;
}

/* The directory set of the batch finished last (n >= 1 records) into `ch` (ctx->ch, or ctx->evq for regk_read_events):
   its distinct parents in parent order, listed (valid, not "/") to drec / dlen and, with `pack`, packed to dbytes /
   doff, the others' first records to unlisted. */
extern "C++" {
namespace {
template <class Dirs>
int children_dirs(regk_ctx *ctx, Dirs &ch, bool pack)
{
    cudaStream_t s = ctx->stream;
    const uint64_t n = ctx->last.n;
    int rc;
    if ((rc = ensure_host(ctx, ch.h_count, CQ_NCOUNTERS * 8)) || (rc = ensure_dev(ctx, ch.count, CQ_NCOUNTERS * 8)))
        return rc;
    unsigned long long *hc = (unsigned long long *)ch.h_count.p;
    ParentParams pp{};
    if ((rc = enqueue_parent_pass(ctx, ch.pass, n, nullptr, &pp)))
        return rc;
    CK(cudaMemcpyAsync(hc, pp.n_unique, 8, cudaMemcpyDeviceToHost, s));
    if ((rc = sync_or_fail(ctx, s, "regk_children_requests")))
        return rc;
    const uint64_t nu = hc[0];
    const uint64_t ntiles = (nu + MK_TILE - 1) / MK_TILE, tt = align16(ntiles * 4), st = (ntiles / SUPER + 1) * 8;
    const size_t totals_bytes = 2 * tt + 2 * st + 16;
    if ((rc = ensure_dev(ctx, ch.totals, totals_bytes)) || (rc = ensure_dev(ctx, ch.unlisted, nu * 8 + 8)) ||
        (rc = ensure_dev(ctx, ch.drec, nu * 8 + 8)) || (rc = ensure_dev(ctx, ch.dlen, nu * 4 + 8)))
        return rc;
    uint8_t *tb = (uint8_t *)ch.totals.p;
    ChDirParams dp{};
    dp.path_bytes = ctx->last.path_bytes;
    dp.path_off = ctx->last.path_off;
    dp.parent_len = pp.parent_len;
    dp.unique_first = pp.unique_first;
    dp.nu = nu;
    dp.tile_a = (uint32_t *)tb;
    dp.tile_b = (uint32_t *)(tb + tt);
    dp.super_a = (unsigned long long *)(tb + 2 * tt);
    dp.super_b = (unsigned long long *)(tb + 2 * tt + st);
    dp.counters = (unsigned long long *)ch.count.p;
    dp.unlisted = (unsigned long long *)ch.unlisted.p;
    dp.dir_rec = (unsigned long long *)ch.drec.p;
    dp.dir_len = (uint32_t *)ch.dlen.p;
    CK(cudaMemsetAsync(tb, 0, totals_bytes, s));
    CK(cudaMemsetAsync(ch.count.p, 0, CQ_NCOUNTERS * 8, s));
    regk_children_dirs_count_kernel<<<(unsigned)ntiles, MK_TILE, 0, s>>>(dp);
    regk_children_dirs_kernel<<<(unsigned)ntiles, MK_TILE, 0, s>>>(dp);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(hc, ch.count.p, CQ_NCOUNTERS * 8, cudaMemcpyDeviceToHost, s));
    if ((rc = sync_or_fail(ctx, s, "regk_children_requests")))
        return rc;
    ch.d = hc[CQ_LISTED];
    ch.n_unlisted = hc[CQ_UNLISTED];
    ch.prefixes = hc[CQ_PREFIXES];
    if (!pack)
        return REGK_OK;
    uint64_t bytes = 0;
    uint32_t launches = 0;
    return pack_strings(ctx, ch.d, ctx->last.path_bytes, ctx->last.path_off, (const unsigned long long *)ch.drec.p,
        (const uint32_t *)ch.dlen.p, ch.totals, ch.dbytes, ch.doff, &bytes, &launches);
}
}  // namespace
}  /* extern "C++" */

int regk_children_requests(regk_ctx *ctx, const regk_jute_opts *o, regk_frames *out)
{
    if (!ctx || !o || !out)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_children_requests: NULL argument");
    memset(out, 0, sizeof *out);
    regk_ctx::Children &ch = ctx->ch;
    if (o->op == REGK_ZK_DELETE) {
        if (o->flags & REGK_ZK_WATCH)
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_children_requests: REGK_ZK_WATCH arms a watch with a read; delete (2) "
                                                   "is a write");
        if (o->group > 65536)
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_children_requests: at most 65536 operations per multi transaction");
        if (ctx->pending)
            return fail(ctx, REGK_ERR_STATE, "regk_children_requests: batches are still in flight; finish them first");
        if (!ch.read)
            return fail(ctx, REGK_ERR_STATE, "regk_children_requests: no stale list on this context; call regk_read_children first");
        CK(cudaSetDevice(ctx->device));
        FrameSrc src{ch.n_stale, (const uint8_t *)ch.sbytes.p, (const unsigned long long *)ch.soff.p, nullptr, nullptr};
        src.who = "regk_children_requests";
        const int rc = frame_requests(ctx, src, o, ch.frames[1], out);
        if (rc == REGK_OK)
            record_framing(ctx->rs.stale, src, o, REGK_ZK_DELETE, o->group != 0, out->n, (const unsigned long long *)ch.stale.p,
                ch.read_gen);
        return rc;
    }
    if (o->op != REGK_ZK_GETCHILDREN)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_children_requests: op %u is not getChildren (8) or delete (2)", o->op);
    if (o->group != 0)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_children_requests: getChildren requests cannot go in a multi transaction "
                                               "(group %u)", o->group);
    if (ctx->pending)
        return fail(ctx, REGK_ERR_STATE, "regk_children_requests: batches are still in flight; finish them first");
    if (!ctx->last.path_off || !ctx->last.path_bytes || ctx->last.n == 0)
        return fail(ctx, REGK_ERR_STATE, "regk_children_requests: no finished batch with a path stream on this context (an "
                                         "empty batch, a REGK_NO_PATH batch or a REGK_JOB_STEP result leaves none)");
    if (ctx->last.alias)
        return fail(ctx, REGK_ERR_STATE, "regk_children_requests: the batch finished last holds alias nodes; their parents are "
                                         "domain directories that hold other services, not service directories");
    if (ctx->last.n >= 0xFFFFFFFEull)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_children_requests: batch too large");
    CK(cudaSetDevice(ctx->device));
    int rc;
    if ((rc = watch_forget_unread(ctx, true, nullptr)))
        return rc;
    ch.framed = false;
    if ((rc = children_dirs(ctx, ch, true)))
        return rc;
    FrameSrc src{ch.d, (const uint8_t *)ch.dbytes.p, (const unsigned long long *)ch.doff.p, nullptr, nullptr};
    src.who = "regk_children_requests";
    if ((rc = frame_requests(ctx, src, o, ch.frames[0], out)))
        return rc;
    ch.framed = true;
    ch.gen = ctx->last.gen;
    ch.n = ctx->last.n;
    ch.xid = o->xid_base;
    ch.keep_drec = (const unsigned long long *)ch.drec.p;
    ch.keep_dlen = (const uint32_t *)ch.dlen.p;
    ch.keep_d = ch.d;
    ch.sub_item = nullptr;
    return watch_framed(ctx, true, o->flags & REGK_ZK_WATCH);
}

static const char *children_reason(uint32_t code)
{
    switch (code) {
    case CH_TRUNC: return "the stream ends inside the frame";
    case CH_BAD_LEN: return "a frame length below 16 (no room for a ReplyHeader)";
    case CH_NEG_XID: return "a negative xid other than -1 (notification) or -2 (ping)";
    case CH_XID_RANGE: return "an xid outside the framed requests";
    case CH_ERR_BODY: return "an error reply with a body";
    case CH_SUCC_LEN: return "a success frame too short for its count";
    case CH_NEG_COUNT: return "a child count below -1";
    case CH_ORDER: return "a reply out of order, or for a directory that already has one";
    case CH_ENT_TRUNC: return "an entry runs past the end of its frame";
    case CH_ENT_EMPTY: return "an entry with an empty name";
    case CH_NAME_SLASH: return "a name holding '/'";
    case CH_NAME_NUL: return "a name holding a NUL byte";
    case CH_NAME_DOT: return "a name that is '.' or '..'";
    case CH_ENT_END: return "the entries end before the frame does";
    default: return "internal error";
    }
}

/* The chain machinery of regk_replies.cuh over the candidates p->word .. p->tile_base already count: compact, J_0 .. J_K
   (2^(K+1) > reach), and the marking from the seeds `seed` enqueues.  Sets p->cand, p->marked, p->C; *j0 = J_0. */
static int chain_pass(regk_ctx *ctx, RepParams *p, uint64_t tiles_s, uint64_t reach, DevBuf &cand, DevBuf &mark,
    DevBuf &jump, const std::function<void(const RepParams &)> &seed, uint32_t **j0, uint32_t *launches, const char *who)
{
    cudaStream_t s = ctx->stream;
    const uint64_t nsup = tiles_s / SUPER + 1;
    std::vector<unsigned long long> sup(nsup, 0);
    CK(cudaMemcpyAsync(sup.data(), p->super_total, nsup * 8, cudaMemcpyDeviceToHost, s));
    int rc;
    if ((rc = sync_or_fail(ctx, s, who)))
        return rc;
    uint64_t C = 0;
    for (unsigned long long v : sup)
        C += v;
    if (C >= 0xFFFFFFFFull)
        return fail(ctx, REGK_ERR_INVALID_ARG, "%s: %llu plausible positions in the stream: must be below 2^32 - 1", who,
            (unsigned long long)C);
    uint32_t K = 0;
    while ((1ull << (K + 1)) <= std::min<uint64_t>(reach, C))
        K++;
    if ((rc = ensure_dev(ctx, cand, C * 8 + 16)) || (rc = ensure_dev(ctx, mark, C + 16)) ||
        (rc = ensure_dev(ctx, jump, (size_t)(K + 1) * C * 4 + 16)))
        return rc;
    p->cand = (unsigned long long *)cand.p;
    p->marked = (uint8_t *)mark.p;
    p->C = C;
    uint32_t *J = (uint32_t *)jump.p;
    *j0 = J;
    if (!C)
        return REGK_OK;
    const unsigned g256 = (unsigned)((C + 255) / 256);
    regk_replies_compact_kernel<<<(unsigned)tiles_s, RP_TILE, 0, s>>>(*p);
    regk_replies_succ_kernel<<<g256, 256, 0, s>>>(*p, J);
    for (uint32_t l = 0; l < K; l++)
        regk_replies_jump_kernel<<<g256, 256, 0, s>>>(J + (size_t)l * C, J + (size_t)(l + 1) * C, C);
    CK(cudaMemsetAsync(p->marked, 0, C, s));
    seed(*p);
    for (uint32_t l = K + 1; l-- > 0;)
        regk_replies_mark_kernel<<<g256, 256, 0, s>>>(*p, J + (size_t)l * C, 0u);
    CK(cudaGetLastError());
    *launches += 2 * K + 4;
    return REGK_OK;
}

int regk_read_children(regk_ctx *ctx, const uint8_t *bytes, uint64_t len, uint64_t start, uint32_t flags, regk_children *out)
{
    const char *who = "regk_read_children";
    if (!ctx || !out)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_children: NULL argument");
    memset(out, 0, sizeof *out);
    regk_ctx::Children &ch = ctx->ch;
    if (ctx->pending)
        return fail(ctx, REGK_ERR_STATE, "regk_read_children: batches are still in flight; finish them first");
    if (!ch.framed)
        return fail(ctx, REGK_ERR_STATE, "regk_read_children: no getChildren framing (regk_children_requests with "
                                         "REGK_ZK_GETCHILDREN) of the batch finished last");
    if (ch.gen != ctx->last.gen || !ctx->last.path_off)
        return fail(ctx, REGK_ERR_STATE, "regk_read_children: a batch finished after the getChildren framing; frame its "
                                         "getChildren requests first");
    if (!bytes && len)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_children: NULL stream of %llu bytes", (unsigned long long)len);
    if (start > len)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_children: start %llu is past the stream's %llu bytes",
            (unsigned long long)start, (unsigned long long)len);
    const bool in_dev = flags & REGK_IN_DEVICE, dev_out = flags & REGK_OUT_DEVICE;
    if (in_dev && ((uintptr_t)bytes & 15u))
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_children: misaligned device stream (16-byte alignment needed)");
    const uint64_t d = ch.d;
    const int32_t xb = ch.xid;
    for (int32_t reserved : {-1, -2})
        if ((uint64_t)((uint32_t)reserved - (uint32_t)xb) < d)
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_children: the framed xids [%d, %d + %llu) cover %d, which ZooKeeper "
                                                   "uses for %s", xb, xb, (unsigned long long)d, reserved,
                        reserved == -1 ? "watch notifications" : "pings");
    if (d >= 0xFFFFFFFFull)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_children: %llu directories: must be below 2^32 - 1", (unsigned long long)d);
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    ch.read = false;
    ch.read_gen++;
    int rc;
    for (Event &ev : ch.ev)
        if ((rc = ensure_event(ctx, ev)))
            return rc;
    const uint8_t *ds = bytes;
    if (!in_dev && len) {
        if ((rc = stage_in(ctx, ch.stream, bytes, len, s)))
            return rc;
        ds = (const uint8_t *)ch.stream.p;
    }
    const uint64_t nblk = (len + 15) / 16, tiles_s = (nblk + RP_TILE - 1) / RP_TILE;
    const size_t totals_bytes = align16(tiles_s * 4) + (tiles_s / SUPER + 1) * 8;
    const size_t d8 = d * 8 + 16, d4 = d * 4 + 16;
    if ((rc = ensure_dev(ctx, ch.word, nblk * 4 + 16)) || (rc = ensure_dev(ctx, ch.ftotals, totals_bytes)) ||
        (rc = ensure_dev(ctx, ch.tile_base, tiles_s * 8 + 16)) || (rc = ensure_dev(ctx, ch.fpos, d8)) ||
        (rc = ensure_dev(ctx, ch.fend, d8)) || (rc = ensure_dev(ctx, ch.err, d4)) || (rc = ensure_dev(ctx, ch.cnt, d4)) ||
        (rc = ensure_dev(ctx, ch.seed_g, d4)) || (rc = ensure_dev(ctx, ch.last_g1, d4)) ||
        (rc = ensure_dev(ctx, ch.name_bad, d4)) || (rc = ensure_dev(ctx, ch.end_pos, d8)) ||
        (rc = ensure_dev(ctx, ch.fault_pos, d8)) || (rc = ensure_dev(ctx, ch.child_off, d8)) ||
        (rc = ensure_host(ctx, ch.h_count, CQ_NCOUNTERS * 8)) || (rc = ensure_dev(ctx, ch.count, CQ_NCOUNTERS * 8)))
        return rc;
    ChParams cp{};
    RepParams &p = cp.r;
    p.s = ds;
    p.len = len;
    p.xid_base = xb;
    p.n = d;
    p.word = (uint32_t *)ch.word.p;
    p.tile_total = (uint32_t *)ch.ftotals.p;
    p.super_total = (unsigned long long *)((uint8_t *)ch.ftotals.p + align16(tiles_s * 4));
    p.tile_base = (unsigned long long *)ch.tile_base.p;
    p.counters = (unsigned long long *)ch.count.p;
    cp.start = start;
    cp.d = d;
    cp.fpos = (unsigned long long *)ch.fpos.p;
    cp.fend = (unsigned long long *)ch.fend.p;
    cp.err = (int32_t *)ch.err.p;
    cp.cnt = (uint32_t *)ch.cnt.p;
    cp.seed_g = (uint32_t *)ch.seed_g.p;
    cp.last_g1 = (uint32_t *)ch.last_g1.p;
    cp.name_bad = (uint32_t *)ch.name_bad.p;
    cp.end_pos = (unsigned long long *)ch.end_pos.p;
    cp.fault_pos = (unsigned long long *)ch.fault_pos.p;
    cp.child_off = (unsigned long long *)ch.child_off.p;
    cp.dir_len = (const uint32_t *)ch.dlen.p;
    unsigned long long *hc = (unsigned long long *)ch.h_count.p;
    CK(cudaMemsetAsync(p.counters, 0, CQ_NCOUNTERS * 8, s));
    CK(cudaMemsetAsync(p.counters + RQ_ERR, 0xFF, 8, s));
    CK(cudaMemsetAsync(p.counters + CQ_ENT_ERR, 0xFF, 8, s));
    CK(cudaMemsetAsync(p.tile_total, 0, totals_bytes, s));
    CK(cudaEventRecord(ch.ev[0], s));
    uint32_t launches = 0;
    /* 1. the frame chain from `start` and the replies of the d directories */
    RepParams pf = p;
    if (d && len) {
        regk_children_cand_kernel<<<(unsigned)tiles_s, RP_TILE, 0, s>>>(cp);
        CK(cudaGetLastError());
        launches++;
        uint32_t *J = nullptr;
        if ((rc = chain_pass(ctx, &pf, tiles_s, ~0ull, ch.cand, ch.mark, ch.jump, [&](const RepParams &q) {
                regk_children_seed_kernel<<<1, 256, 0, s>>>(q, nullptr, nullptr, 1, start);
            }, &J, &launches, who)))
            return rc;
        if (pf.C) {
            const uint64_t tiles_c = (pf.C + RP_TILE - 1) / RP_TILE;
            const size_t t2 = align16(tiles_c * 4) + (tiles_c / SUPER + 1) * 8;
            if ((rc = ensure_dev(ctx, ch.totals2, t2)))
                return rc;
            cp.r = pf;
            cp.r.tile_total = (uint32_t *)ch.totals2.p;
            cp.r.super_total = (unsigned long long *)((uint8_t *)ch.totals2.p + align16(tiles_c * 4));
            CK(cudaMemsetAsync(ch.totals2.p, 0, t2, s));
            regk_replies_chain_count_kernel<<<(unsigned)tiles_c, RP_TILE, 0, s>>>(cp.r);
            regk_children_chain_kernel<<<(unsigned)tiles_c, RP_TILE, 0, s>>>(cp);
            CK(cudaGetLastError());
            launches += 3;
        }
    }
    CK(cudaMemcpyAsync(hc, p.counters, CQ_NCOUNTERS * 8, cudaMemcpyDeviceToHost, s));
    if ((rc = sync_or_fail(ctx, s, who)))
        return rc;
    const uint64_t frame_err_k = hc[RQ_ERR] != ~0ull ? hc[RQ_ERR] >> 8 : d;
    const uint64_t d_eff = std::min<uint64_t>(std::min<uint64_t>(frame_err_k, hc[RQ_NREP]), d);
    const uint64_t n_skipped = hc[RQ_SKIP], n_found = hc[RQ_FOUND], n_missing = hc[RQ_MISSING], n_error = hc[RQ_ERROR];
    const uint64_t consumed = d ? hc[RQ_CONSUMED] : start;
    /* 2. the entry chains inside the success frames of the first d_eff replies; every frame's entries against its count */
    uint64_t ne = 0;
    if (d_eff) {
        cp.d_eff = d_eff;
        if ((rc = ensure_dev(ctx, ch.eword, nblk * 4 + 16)) || (rc = ensure_dev(ctx, ch.etotals, totals_bytes)) ||
            (rc = ensure_dev(ctx, ch.etile_base, tiles_s * 8 + 16)))
            return rc;
        RepParams pe = p;
        pe.word = (uint32_t *)ch.eword.p;
        pe.tile_total = (uint32_t *)ch.etotals.p;
        pe.super_total = (unsigned long long *)((uint8_t *)ch.etotals.p + align16(tiles_s * 4));
        pe.tile_base = (unsigned long long *)ch.etile_base.p;
        CK(cudaMemsetAsync(pe.tile_total, 0, totals_bytes, s));
        CK(cudaMemsetAsync(cp.seed_g, 0xFF, d_eff * 4, s));
        CK(cudaMemsetAsync(cp.name_bad, 0xFF, d_eff * 4, s));
        CK(cudaMemsetAsync(cp.last_g1, 0, d_eff * 4, s));
        cp.r = pe;
        regk_children_ent_cand_kernel<<<(unsigned)tiles_s, RP_TILE, 0, s>>>(cp);
        CK(cudaGetLastError());
        launches++;
        uint32_t *J = nullptr;
        const unsigned gd = (unsigned)((d_eff + 255) / 256);
        if ((rc = chain_pass(ctx, &pe, tiles_s, hc[CQ_MAXC] + 1, ch.ecand, ch.emark, ch.ejump, [&](const RepParams &q) {
                regk_children_seed_kernel<<<gd, 256, 0, s>>>(q, cp.fpos, cp.cnt, d_eff, 24ull);
            }, &J, &launches, who)))
            return rc;
        const uint64_t Ce = pe.C;
        if ((rc = ensure_dev(ctx, ch.ent_pos, Ce * 8 + 16)) || (rc = ensure_dev(ctx, ch.ent_nlen, Ce * 4 + 16)) ||
            (rc = ensure_dev(ctx, ch.ent_k, Ce * 4 + 16)) || (rc = ensure_dev(ctx, ch.ent_plen, Ce * 4 + 16)))
            return rc;
        cp.j0 = J;
        cp.ent_pos = (unsigned long long *)ch.ent_pos.p;
        cp.ent_nlen = (uint32_t *)ch.ent_nlen.p;
        cp.ent_k = (uint32_t *)ch.ent_k.p;
        cp.ent_plen = (uint32_t *)ch.ent_plen.p;
        cp.r = pe;
        if (Ce) {
            const uint64_t tiles_e = (Ce + RP_TILE - 1) / RP_TILE;
            const size_t t2 = align16(tiles_e * 4) + (tiles_e / SUPER + 1) * 8;
            if ((rc = ensure_dev(ctx, ch.etotals2, t2)))
                return rc;
            cp.r.tile_total = (uint32_t *)ch.etotals2.p;
            cp.r.super_total = (unsigned long long *)((uint8_t *)ch.etotals2.p + align16(tiles_e * 4));
            CK(cudaMemsetAsync(ch.etotals2.p, 0, t2, s));
            regk_children_ent_count_kernel<<<(unsigned)tiles_e, RP_TILE, 0, s>>>(cp.r);
            regk_children_ent_kernel<<<(unsigned)tiles_e, RP_TILE, 0, s>>>(cp);
            launches += 2;
        }
        regk_children_ent_frame_kernel<<<gd, 256, 0, s>>>(cp);
        CK(cudaGetLastError());
        launches++;
        CK(cudaMemcpyAsync(hc, p.counters, CQ_NCOUNTERS * 8, cudaMemcpyDeviceToHost, s));
        if ((rc = sync_or_fail(ctx, s, who)))
            return rc;
        ne = hc[CQ_NENT];
    }
    /* refusals: the first fault a front-to-back reader meets - an entry fault of a frame before any frame fault */
    if (hc[CQ_ENT_ERR] != ~0ull) {
        const uint64_t k = hc[CQ_ENT_ERR] >> 8;
        const uint32_t code = (uint32_t)(hc[CQ_ENT_ERR] & 0xFF);
        unsigned long long at[2] = {0, 0};
        CK(cudaMemcpyAsync(&at[0], cp.fault_pos + k, 8, cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(&at[1], cp.fpos + k, 8, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_children: byte %llu: %s (entry of the reply frame at byte %llu); "
                                               "expected the reply to directory %llu (xid %d)", at[0], children_reason(code), at[1],
                    (unsigned long long)k, (int32_t)((uint32_t)xb + (uint32_t)k));
    }
    if (hc[RQ_ERR] != ~0ull) {
        const uint64_t k = hc[RQ_ERR] >> 8;
        const uint32_t code = (uint32_t)(hc[RQ_ERR] & 0xFF);
        unsigned long long pos = 0;
        CK(cudaMemcpyAsync(&pos, cp.fpos + k, 8, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_children: byte %llu: %s; expected the reply to directory %llu (xid %d)",
            pos, children_reason(code), (unsigned long long)k, (int32_t)((uint32_t)xb + (uint32_t)k));
    }
    if (hc[RQ_NREP] < d) {
        /* the chain stops before the d-th reply: the frame check where it stops names the reason */
        uint64_t stop = start;
        if (pf.C) {
            regk_replies_stop_kernel<<<(unsigned)((pf.C + 255) / 256), 256, 0, s>>>(pf);
            CK(cudaGetLastError());
            CK(cudaMemcpyAsync(hc + RQ_STOP, p.counters + RQ_STOP, 8, cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
            stop = std::max<uint64_t>(stop, hc[RQ_STOP]);
        }
        const uint64_t done = hc[RQ_NREP];
        uint8_t head[24] = {0};
        const uint64_t avail = len - stop, take = std::min<uint64_t>(avail, sizeof head);
        if (take) {
            CK(cudaMemcpyAsync(head, ds + stop, take, cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
        }
        ChildHead h;
        const uint32_t code = children_head(head, avail, xb, d, &h);
        const int32_t want = (int32_t)((uint32_t)xb + (uint32_t)done);
        if (code == CH_TRUNC)
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_children: byte %llu: the stream ends before the reply to directory "
                                                   "%llu (xid %d) is complete; %llu of %llu replies complete",
                        (unsigned long long)stop, (unsigned long long)done, want, (unsigned long long)done, (unsigned long long)d);
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_children: byte %llu: %s (len %d, xid %d); expected the reply to "
                                               "directory %llu (xid %d)", (unsigned long long)stop,
                    code ? children_reason(code) : "internal error", h.len, h.xid, (unsigned long long)done, want);
    }
    if (ne >= 0xFFFFFFFFull)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_children: %llu children: must be below 2^32 - 1", (unsigned long long)ne);
    if ((rc = ensure_dev(ctx, ch.child_off, d * 8 + 16)))
        return rc;
    CK(cudaMemcpyAsync(cp.child_off + d, &ne, 8, cudaMemcpyHostToDevice, s));
    /* 3. the listing paths */
    uint64_t lst_total = 0;
    {
        const uint64_t gt = (ne + MK_TILE - 1) / MK_TILE;
        if ((rc = ensure_dev(ctx, ch.gtotals, gt * 8 + (gt / SUPER + 1) * 8 + 16)) ||
            (rc = ensure_dev(ctx, ch.lst_off, (ne + 1) * 8)) || (rc = ensure_dev(ctx, ch.lst_zero, (ne + 1) * 8)))
            return rc;
        CK(cudaMemsetAsync(ch.lst_zero.p, 0, (ne + 1) * 8, s));
        if (ne) {
            MkGatherParams gp{};
            gp.n_dirs = ne;
            gp.dir_len = cp.ent_plen;
            gp.tile_total = (unsigned long long *)ch.gtotals.p;
            gp.super_total = gp.tile_total + gt;
            CK(cudaMemsetAsync(gp.super_total, 0, (gt / SUPER + 1) * 8, s));
            regk_mkdirp_len_kernel<<<(unsigned)gt, MK_TILE, 0, s>>>(gp);
            std::vector<unsigned long long> gs(gt / SUPER + 1);
            CK(cudaMemcpyAsync(gs.data(), gp.super_total, gs.size() * 8, cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
            for (unsigned long long v : gs)
                lst_total += v;
            if ((rc = ensure_dev(ctx, ch.lst_bytes, lst_total + 16)))
                return rc;
            ChGatherParams g{};
            g.n = ne;
            g.tile_total = gp.tile_total;
            g.super_total = gp.super_total;
            g.ent_k = cp.ent_k;
            g.ent_nlen = cp.ent_nlen;
            g.ent_plen = cp.ent_plen;
            g.ent_pos = cp.ent_pos;
            g.dir_bytes = (const uint8_t *)ch.dbytes.p;
            g.dir_off = (const unsigned long long *)ch.doff.p;
            g.s = ds;
            g.out_bytes = (uint8_t *)ch.lst_bytes.p;
            g.out_off = (unsigned long long *)ch.lst_off.p;
            regk_children_gather_kernel<<<(unsigned)gt, MK_TILE, 0, s>>>(g);
            CK(cudaGetLastError());
            launches += 2;
        } else {
            if ((rc = ensure_dev(ctx, ch.lst_bytes, 16)))
                return rc;
            CK(cudaMemsetAsync(ch.lst_off.p, 0, 8, s));
        }
    }
    /* 4. the keep table, every listing path's class, the stale list and its packed paths */
    uint64_t n_stale = 0;
    const uint64_t tiles_l = (ne + MK_TILE - 1) / MK_TILE;
    if ((rc = ensure_dev(ctx, ch.cls, ne + 16)) || (rc = ensure_dev(ctx, ch.stale, ne * 8 + 16)) ||
        (rc = ensure_dev(ctx, ch.stale_len, ne * 4 + 16)))
        return rc;
    if (ne) {
        const uint64_t entries = ch.n + ch.prefixes;
        uint64_t slots = 1024;
        while (slots < 2 * entries)
            slots <<= 1;
        if (slots > (1ull << 32))
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_children: %llu paths and directories are too many for one table",
                (unsigned long long)entries);
        const size_t st_bytes = align16(tiles_l * 4) + (tiles_l / SUPER + 1) * 8;
        if ((rc = ensure_dev(ctx, ch.table, slots * 8)) || (rc = ensure_dev(ctx, ch.stotals, st_bytes)))
            return rc;
        ChKeepParams kp{};
        kp.path_bytes = ctx->last.path_bytes;
        kp.path_off = ctx->last.path_off;
        kp.n = ch.n;
        kp.dir_rec = ch.keep_drec;
        kp.dir_len = ch.keep_dlen;
        kp.d = ch.keep_d;
        kp.table = (unsigned long long *)ch.table.p;
        kp.mask = (uint32_t)(slots - 1);
        kp.lst_bytes = (const uint8_t *)ch.lst_bytes.p;
        kp.lst_off = (const unsigned long long *)ch.lst_off.p;
        kp.n_children = ne;
        kp.cls = (uint8_t *)ch.cls.p;
        kp.tile_total = (uint32_t *)ch.stotals.p;
        kp.super_total = (unsigned long long *)((uint8_t *)ch.stotals.p + align16(tiles_l * 4));
        kp.stale = (unsigned long long *)ch.stale.p;
        kp.stale_len = (uint32_t *)ch.stale_len.p;
        kp.counters = p.counters;
        CK(cudaMemsetAsync(kp.table, 0, slots * 8, s));
        CK(cudaMemsetAsync(ch.stotals.p, 0, st_bytes, s));
        regk_children_keep_paths_kernel<<<(unsigned)((ch.n + 255) / 256), 256, 0, s>>>(kp);
        if (kp.d)
            regk_children_keep_dirs_kernel<<<(unsigned)((kp.d + 255) / 256), 256, 0, s>>>(kp);
        regk_children_probe_kernel<<<(unsigned)tiles_l, MK_TILE, 0, s>>>(kp);
        regk_children_stale_kernel<<<(unsigned)tiles_l, MK_TILE, 0, s>>>(kp);
        CK(cudaGetLastError());
        launches += kp.d ? 4 : 3;
        CK(cudaMemcpyAsync(hc + CQ_STALE, p.counters + CQ_STALE, 8, cudaMemcpyDeviceToHost, s));
        if ((rc = sync_or_fail(ctx, s, who)))
            return rc;
        n_stale = hc[CQ_STALE];
    }
    uint64_t stale_bytes = 0;
    if ((rc = pack_strings(ctx, n_stale, (const uint8_t *)ch.lst_bytes.p, (const unsigned long long *)ch.lst_off.p,
             (const unsigned long long *)ch.stale.p, (const uint32_t *)ch.stale_len.p, ch.gtotals, ch.sbytes, ch.soff,
             &stale_bytes, &launches)))
        return rc;
    /* the directory set this read answers, kept with the read (a later framing rebuilds the framing's own) */
    const uint64_t nun = ch.n_unlisted;
    if ((rc = ensure_dev(ctx, ch.r_drec, d * 8 + 8)) || (rc = ensure_dev(ctx, ch.r_dlen, d * 4 + 8)) ||
        (rc = ensure_dev(ctx, ch.r_unlisted, nun * 8 + 8)))
        return rc;
    if (d) {
        CK(cudaMemcpyAsync(ch.r_drec.p, ch.drec.p, d * 8, cudaMemcpyDeviceToDevice, s));
        CK(cudaMemcpyAsync(ch.r_dlen.p, ch.dlen.p, d * 4, cudaMemcpyDeviceToDevice, s));
    }
    if (nun)
        CK(cudaMemcpyAsync(ch.r_unlisted.p, ch.unlisted.p, nun * 8, cudaMemcpyDeviceToDevice, s));
    CK(cudaEventRecord(ch.ev[1], s));
    if ((rc = sync_or_fail(ctx, s, who)))
        return rc;
    float ms = 0;
    cudaEventElapsedTime(&ms, ch.ev[0], ch.ev[1]);
    const void *src[7] = {ch.r_drec.p, ch.r_dlen.p, ch.err.p, ch.child_off.p, ch.cls.p, ch.stale.p, ch.r_unlisted.p};
    if (!dev_out) {
        HostBuf *hb[7] = {&ch.h_drec, &ch.h_dlen, &ch.h_err, &ch.h_child_off, &ch.h_cls, &ch.h_stale, &ch.h_unlisted};
        const size_t sz[7] = {d * 8, d * 4, d * 4, (d + 1) * 8, ne, n_stale * 8, nun * 8};
        for (int k = 0; k < 7; k++) {
            if ((rc = to_host(ctx, *hb[k], src[k], sz[k], s)))
                return rc;
            src[k] = hb[k]->p;
        }
        CK(cudaStreamSynchronize(s));
    }
    if ((rc = watch_read(ctx, true, (const int32_t *)ch.err.p, d, ch.sub_item, ch.keep_d)))
        return rc;
    ch.read = true;
    ch.n_stale = n_stale;
    out->n_dirs = d;
    out->n_children = ne;
    out->n_stale = n_stale;
    out->n_found = n_found;
    out->n_missing = n_missing;
    out->n_error = n_error;
    out->n_skipped = n_skipped;
    out->consumed = consumed;
    out->n_unlisted = nun;
    out->flags = dev_out ? REGK_OUT_DEVICE : 0;
    out->launches = launches;
    out->dir_rec = (const uint64_t *)src[0];
    out->dir_len = (const uint32_t *)src[1];
    out->err = (const int32_t *)src[2];
    out->child_off = (const uint64_t *)src[3];
    out->cls = (const uint8_t *)src[4];
    out->stale = (const uint64_t *)src[5];
    out->unlisted = (const uint64_t *)src[6];
    out->listing.n = ne;
    out->listing.flags = REGK_IN_DEVICE;
    out->listing.host_nodes = 1;
    out->listing.path_total = lst_total;
    out->listing.json_total = 0;
    out->listing.path_bytes = (const uint8_t *)ch.lst_bytes.p;
    out->listing.path_off = (const uint64_t *)ch.lst_off.p;
    out->listing.json_bytes = (const uint8_t *)ch.lst_bytes.p;
    out->listing.json_off = (const uint64_t *)ch.lst_zero.p;
    out->kernel_ms = ms;
    return REGK_OK;
}

static const char *results_reason(uint32_t code)
{
    switch (code) {
    case RS_TRUNC: return "the stream ends inside the frame";
    case RS_BAD_LEN: return "a frame length below 16 (no room for a ReplyHeader)";
    case RS_NEG_XID: return "a negative xid other than -1 (notification) or -2 (ping)";
    case RS_XID_RANGE: return "an xid outside the framed requests";
    case RS_ERR_BODY: return "an error reply with a body";
    case RS_SUCC_LEN: return "a success length that fits neither outcome of the frame";
    case RS_ORDER: return "a reply out of order, or for a frame that already has one";
    case RS_OP_TYPE: return "a MultiHeader of the wrong type, done flag or err";
    case RS_PATH_ECHO: return "a create path echo that differs from the framed path";
    case RS_STAT_LEN: return "Stat.dataLength differs from the framed data's length";
    case RS_ERR_RESULT: return "an ErrorResult whose two codes differ";
    case RS_ERR_SEQ: return "ErrorResults out of the 0 / failing code / -2 order";
    case RS_CLOSE: return "the multi's closing MultiHeader{-1, true, -1} is missing";
    case RS_NO_FAILURE: return "a rolled-back multi with no nonzero ErrorResult";
    default: return "internal error";
    }
}

int regk_read_results(regk_ctx *ctx, const uint8_t *bytes, uint64_t len, uint64_t start, const regk_results_opts *o,
    regk_results *out)
{
    const char *who = "regk_read_results";
    if (!ctx || !o || !out)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_results: NULL argument");
    memset(out, 0, sizeof *out);
    regk_ctx::Results &rs = ctx->rs;
    const regk_ctx::ResDesc *dsc = nullptr;
    uint64_t gen = 0;
    const char *changed = "";
    switch (o->source) {
    case REGK_RES_BATCH:
        dsc = &rs.batch, gen = ctx->last.gen, changed = "a batch finished";
        break;
    case REGK_RES_MKDIRP:
        dsc = &rs.mkdirp, gen = ctx->mk.gen, changed = "regk_mkdirp_dirs ran";
        break;
    case REGK_RES_RECONCILE: {
        const int q = o->op == REGK_ZK_CREATE ? 0 : o->op == REGK_ZK_DELETE ? 1 : o->op == REGK_ZK_SETDATA ? 2
                    : o->op == REGK_ZK_REPLACE ? 3 : -1;
        if (q < 0)
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_results: op %u is not create (1), delete (2), setData (5) or "
                                                   "replace (256)", o->op);
        dsc = &rs.rec[q], gen = ctx->rc.gen, changed = "a reconcile ran";
        break;
    }
    case REGK_RES_STALE:
        dsc = &rs.stale, gen = ctx->ch.read_gen, changed = "regk_read_children ran";
        break;
    default:
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_results: source %u is not REGK_RES_BATCH (1), _MKDIRP (2), "
                                               "_RECONCILE (3) or _STALE (4)", o->source);
    }
    if (ctx->pending)
        return fail(ctx, REGK_ERR_STATE, "regk_read_results: batches are still in flight; finish them first");
    if (!dsc->valid)
        return fail(ctx, REGK_ERR_STATE, "regk_read_results: no write framing of source %u on this context", o->source);
    if (dsc->gen != gen)
        return fail(ctx, REGK_ERR_STATE, "regk_read_results: %s after the framing; its paths are gone, frame the writes again",
            changed);
    if (!bytes && len)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_results: NULL stream of %llu bytes", (unsigned long long)len);
    if (start > len)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_results: start %llu is past the stream's %llu bytes",
            (unsigned long long)start, (unsigned long long)len);
    const bool in_dev = o->flags & REGK_IN_DEVICE, dev_out = o->flags & REGK_OUT_DEVICE;
    if (in_dev && ((uintptr_t)bytes & 15u))
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_results: misaligned device stream (16-byte alignment needed)");
    const ResFraming &f = dsc->f;
    const uint64_t F = f.frames, n = f.entries;
    const int32_t xb = f.xid_base;
    for (int32_t reserved : {-1, -2})
        if ((uint64_t)((uint32_t)reserved - (uint32_t)xb) < F)
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_results: the framed xids [%d, %d + %llu) cover %d, which ZooKeeper "
                                                   "uses for %s", xb, xb, (unsigned long long)F, reserved,
                        reserved == -1 ? "watch notifications" : "pings");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    int rc;
    for (Event &ev : rs.ev)
        if ((rc = ensure_event(ctx, ev)))
            return rc;
    const uint8_t *ds = bytes;
    if (!in_dev && len) {
        if ((rc = stage_in(ctx, rs.stream, bytes, len, s)))
            return rc;
        ds = (const uint8_t *)rs.stream.p;
    }
    const uint64_t nblk = (len + 15) / 16, tiles_s = (nblk + RP_TILE - 1) / RP_TILE;
    const uint64_t tiles_e = (n + RP_TILE - 1) / RP_TILE;
    const size_t totals_bytes = align16(tiles_s * 4) + (tiles_s / SUPER + 1) * 8;
    const size_t tt = align16(tiles_e * 4), st = (tiles_e / SUPER + 1) * 8, ltotals_bytes = 2 * tt + 2 * st;
    if ((rc = ensure_dev(ctx, rs.word, nblk * 4 + 16)) || (rc = ensure_dev(ctx, rs.totals, totals_bytes)) ||
        (rc = ensure_dev(ctx, rs.tile_base, tiles_s * 8 + 16)) || (rc = ensure_dev(ctx, rs.fpos, F * 8 + 16)) ||
        (rc = ensure_dev(ctx, rs.ferr, F * 4 + 16)) || (rc = ensure_dev(ctx, rs.err, n * 4 + 16)) ||
        (rc = ensure_dev(ctx, rs.cls, n + 16)) || (rc = ensure_dev(ctx, rs.ver, n * 4 + 16)) ||
        (rc = ensure_dev(ctx, rs.subject, n * 8 + 16)) || (rc = ensure_dev(ctx, rs.fault_at, n * 8 + 16)) ||
        (rc = ensure_dev(ctx, rs.failed, n * 8 + 16)) || (rc = ensure_dev(ctx, rs.aborted, n * 8 + 16)) ||
        (rc = ensure_dev(ctx, rs.ltotals, ltotals_bytes + 16)) || (rc = ensure_host(ctx, rs.h_count, RS_NCOUNTERS * 8)) ||
        (rc = ensure_dev(ctx, rs.count, RS_NCOUNTERS * 8)))
        return rc;
    ResParams rp{};
    RepParams &p = rp.r;
    p.s = ds;
    p.len = len;
    p.xid_base = xb;
    p.n = F;
    p.word = (uint32_t *)rs.word.p;
    p.tile_total = (uint32_t *)rs.totals.p;
    p.super_total = (unsigned long long *)((uint8_t *)rs.totals.p + align16(tiles_s * 4));
    p.tile_base = (unsigned long long *)rs.tile_base.p;
    p.counters = (unsigned long long *)rs.count.p;
    rp.f = f;
    rp.start = start;
    rp.tol = dsc->tol;
    rp.fpos = (unsigned long long *)rs.fpos.p;
    rp.ferr = (int32_t *)rs.ferr.p;
    rp.subject_in = dsc->subject;
    rp.err = (int32_t *)rs.err.p;
    rp.cls = (uint8_t *)rs.cls.p;
    rp.ver = (int32_t *)rs.ver.p;
    rp.subject = (unsigned long long *)rs.subject.p;
    rp.fault_at = (unsigned long long *)rs.fault_at.p;
    uint8_t *lt = (uint8_t *)rs.ltotals.p;
    rp.tile_a = (uint32_t *)lt;
    rp.tile_b = (uint32_t *)(lt + tt);
    rp.super_a = (unsigned long long *)(lt + 2 * tt);
    rp.super_b = (unsigned long long *)(lt + 2 * tt + st);
    rp.failed = (unsigned long long *)rs.failed.p;
    rp.aborted = (unsigned long long *)rs.aborted.p;
    unsigned long long *hc = (unsigned long long *)rs.h_count.p;
    CK(cudaMemsetAsync(p.counters, 0, RS_NCOUNTERS * 8, s));
    CK(cudaMemsetAsync(p.counters + RQ_ERR, 0xFF, 8, s));
    CK(cudaMemsetAsync(p.counters + RS_ENT_ERR, 0xFF, 8, s));
    CK(cudaMemsetAsync(p.tile_total, 0, totals_bytes, s));
    CK(cudaEventRecord(rs.ev[0], s));
    uint32_t launches = 0;
    /* 1. the frame chain from `start` and the replies of the F frames */
    RepParams pf = p;
    if (F && len) {
        regk_results_cand_kernel<<<(unsigned)tiles_s, RP_TILE, 0, s>>>(rp);
        CK(cudaGetLastError());
        launches++;
        uint32_t *J = nullptr;
        if ((rc = chain_pass(ctx, &pf, tiles_s, ~0ull, rs.cand, rs.mark, rs.jump, [&](const RepParams &q) {
                regk_children_seed_kernel<<<1, 256, 0, s>>>(q, nullptr, nullptr, 1, start);
            }, &J, &launches, who)))
            return rc;
        if (pf.C) {
            const uint64_t tiles_c = (pf.C + RP_TILE - 1) / RP_TILE;
            const size_t t2 = align16(tiles_c * 4) + (tiles_c / SUPER + 1) * 8;
            if ((rc = ensure_dev(ctx, rs.totals2, t2)))
                return rc;
            rp.r = pf;
            rp.r.tile_total = (uint32_t *)rs.totals2.p;
            rp.r.super_total = (unsigned long long *)((uint8_t *)rs.totals2.p + align16(tiles_c * 4));
            CK(cudaMemsetAsync(rs.totals2.p, 0, t2, s));
            regk_replies_chain_count_kernel<<<(unsigned)tiles_c, RP_TILE, 0, s>>>(rp.r);
            regk_results_chain_kernel<<<(unsigned)tiles_c, RP_TILE, 0, s>>>(rp);
            CK(cudaGetLastError());
            launches += 3;
        }
    }
    CK(cudaMemcpyAsync(hc, p.counters, RS_NCOUNTERS * 8, cudaMemcpyDeviceToHost, s));
    if ((rc = sync_or_fail(ctx, s, who)))
        return rc;
    const uint64_t frame_err_k = hc[RQ_ERR] != ~0ull ? hc[RQ_ERR] >> 8 : F;
    const uint64_t f_eff = std::min<uint64_t>(std::min<uint64_t>(frame_err_k, hc[RQ_NREP]), F);
    const uint64_t n_skipped = hc[RQ_SKIP], consumed = F ? hc[RQ_CONSUMED] : start;
    /* 2. every entry of the frames before the first frame fault, and the FAILED / ABORTED lists */
    rp.n_eff = std::min<uint64_t>(f_eff * f.group, n);
    if (rp.n_eff) {
        const unsigned te = (unsigned)((rp.n_eff + RP_TILE - 1) / RP_TILE);
        CK(cudaMemsetAsync(lt, 0, ltotals_bytes, s));
        regk_results_entry_kernel<<<te, RP_TILE, 0, s>>>(rp);
        regk_results_list_kernel<<<te, RP_TILE, 0, s>>>(rp);
        CK(cudaGetLastError());
        launches += 2;
        CK(cudaMemcpyAsync(hc, p.counters, RS_NCOUNTERS * 8, cudaMemcpyDeviceToHost, s));
        if ((rc = sync_or_fail(ctx, s, who)))
            return rc;
    }
    /* refusals: the first fault a front-to-back reader meets - an entry fault of a frame before any frame fault */
    if (hc[RS_ENT_ERR] != ~0ull) {
        const uint64_t e = hc[RS_ENT_ERR] >> 8, k = e / f.group;
        const uint32_t code = (uint32_t)(hc[RS_ENT_ERR] & 0xFF);
        unsigned long long at[2] = {0, 0};
        CK(cudaMemcpyAsync(&at[0], rp.fault_at + e, 8, cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(&at[1], rp.fpos + k, 8, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_results: byte %llu: %s (entry %llu of the reply frame at byte %llu); "
                                               "expected the reply to frame %llu (xid %d)", at[0], results_reason(code),
                    (unsigned long long)e, at[1], (unsigned long long)k, (int32_t)((uint32_t)xb + (uint32_t)k));
    }
    if (hc[RQ_ERR] != ~0ull) {
        const uint64_t k = hc[RQ_ERR] >> 8;
        const uint32_t code = (uint32_t)(hc[RQ_ERR] & 0xFF);
        unsigned long long pos = 0;
        CK(cudaMemcpyAsync(&pos, rp.fpos + k, 8, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_results: byte %llu: %s; expected the reply to frame %llu (xid %d)",
            pos, results_reason(code), (unsigned long long)k, (int32_t)((uint32_t)xb + (uint32_t)k));
    }
    if (hc[RQ_NREP] < F) {
        /* the chain stops before the last reply: the plausibility test where it stops names the reason */
        uint64_t stop = start;
        if (pf.C) {
            regk_replies_stop_kernel<<<(unsigned)((pf.C + 255) / 256), 256, 0, s>>>(pf);
            CK(cudaGetLastError());
            CK(cudaMemcpyAsync(hc + RQ_STOP, p.counters + RQ_STOP, 8, cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
            stop = std::max<uint64_t>(stop, hc[RQ_STOP]);
        }
        const uint64_t done = hc[RQ_NREP];
        uint8_t head[20] = {0};
        const uint64_t avail = len - stop, take = std::min<uint64_t>(avail, sizeof head);
        if (take) {
            CK(cudaMemcpyAsync(head, ds + stop, take, cudaMemcpyDeviceToHost, s));
            regk_results_head_kernel<<<1, 1, 0, s>>>(rp, stop);
            CK(cudaGetLastError());
            CK(cudaMemcpyAsync(hc + RQ_M, p.counters + RQ_M, 8, cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
        }
        const int32_t want = (int32_t)((uint32_t)xb + (uint32_t)done);
        const bool trunc = avail < 4 || ((int32_t)be32_at(head) >= 16 && (uint64_t)(int32_t)be32_at(head) + 4u > avail);
        if (trunc)
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_results: byte %llu: the stream ends before the reply to frame %llu "
                                                   "(xid %d) is complete; %llu of %llu replies complete",
                        (unsigned long long)stop, (unsigned long long)done, want, (unsigned long long)done, (unsigned long long)F);
        const uint32_t code = (uint32_t)hc[RQ_M];
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_results: byte %llu: %s (len %d, xid %d); expected the reply to frame "
                                               "%llu (xid %d)", (unsigned long long)stop, code ? results_reason(code) : "internal error",
                    (int32_t)be32_at(head), take >= 8 ? (int32_t)be32_at(head + 4) : 0, (unsigned long long)done, want);
    }
    CK(cudaEventRecord(rs.ev[1], s));
    if ((rc = sync_or_fail(ctx, s, who)))
        return rc;
    float ms = 0;
    cudaEventElapsedTime(&ms, rs.ev[0], rs.ev[1]);
    const uint64_t n_failed = hc[RS_NFAILED], n_aborted = hc[RS_NABORTED];
    const void *src[7] = {rs.ferr.p, rs.err.p, rs.cls.p, rs.ver.p, rs.subject.p, rs.failed.p, rs.aborted.p};
    if (!dev_out) {
        HostBuf *hb[7] = {&rs.h_ferr, &rs.h_err, &rs.h_cls, &rs.h_ver, &rs.h_subject, &rs.h_failed, &rs.h_aborted};
        const size_t sz[7] = {F * 4, n * 4, n, n * 4, n * 8, n_failed * 8, n_aborted * 8};
        for (int k = 0; k < 7; k++) {
            if ((rc = to_host(ctx, *hb[k], src[k], sz[k], s)))
                return rc;
            src[k] = hb[k]->p;
        }
        CK(cudaStreamSynchronize(s));
    }
    out->n_frames = F;
    out->n_entries = n;
    out->n_done = hc[RS_NDONE];
    out->n_failed = n_failed;
    out->n_aborted = n_aborted;
    out->n_skipped = n_skipped;
    out->consumed = consumed;
    out->flags = dev_out ? REGK_OUT_DEVICE : 0;
    out->launches = launches;
    out->frame_err = (const int32_t *)src[0];
    out->err = (const int32_t *)src[1];
    out->cls = (const uint8_t *)src[2];
    out->version = (const int32_t *)src[3];
    out->subject = (const uint64_t *)src[4];
    out->failed = (const uint64_t *)src[5];
    out->aborted = (const uint64_t *)src[6];
    out->kernel_ms = ms;
    return REGK_OK;
}

static const char *stats_reason(uint32_t code)
{
    switch (code) {
    case ST_TRUNC: return "the stream ends inside the frame";
    case ST_BAD_LEN: return "a frame length below 16 (no room for a ReplyHeader)";
    case ST_NEG_XID: return "a negative xid other than -1 (notification) or -2 (ping)";
    case ST_XID_RANGE: return "an xid outside the framed requests";
    case ST_ERR_BODY: return "an error reply with a body";
    case ST_SUCC_LEN: return "a success frame whose length is not 84 (ReplyHeader + Stat)";
    case ST_ORDER: return "a reply out of order, or for a record that already has one";
    case ST_NEG_DLEN: return "a negative Stat.dataLength";
    default: return "internal error";
    }
}

int regk_read_stats(regk_ctx *ctx, const uint8_t *bytes, uint64_t len, uint64_t start, uint32_t flags, regk_stats *out)
{
    const char *who = "regk_read_stats";
    if (!ctx || !out)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_stats: NULL argument");
    memset(out, 0, sizeof *out);
    regk_ctx::Stats &sq = ctx->sq;
    if (ctx->pending)
        return fail(ctx, REGK_ERR_STATE, "regk_read_stats: batches are still in flight; finish them first");
    if (!ctx->ex_valid)
        return fail(ctx, REGK_ERR_STATE, "regk_read_stats: no exists framing (regk_jute_requests with REGK_ZK_EXISTS) of the "
                                         "batch finished last");
    if (ctx->ex_gen != ctx->last.gen || !ctx->last.path_off)
        return fail(ctx, REGK_ERR_STATE, "regk_read_stats: a batch finished after the exists framing; frame its exists "
                                         "requests first");
    if (!bytes && len)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_stats: NULL stream of %llu bytes", (unsigned long long)len);
    if (start > len)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_stats: start %llu is past the stream's %llu bytes",
            (unsigned long long)start, (unsigned long long)len);
    const bool in_dev = flags & REGK_IN_DEVICE, dev_out = flags & REGK_OUT_DEVICE;
    if (in_dev && ((uintptr_t)bytes & 15u))
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_stats: misaligned device stream (16-byte alignment needed)");
    const uint64_t n = ctx->ex_n;
    const int32_t xb = ctx->ex_xid;
    for (int32_t reserved : {-1, -2})
        if ((uint64_t)((uint32_t)reserved - (uint32_t)xb) < n)
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_stats: the framed xids [%d, %d + %llu) cover %d, which ZooKeeper "
                                                   "uses for %s", xb, xb, (unsigned long long)n, reserved,
                        reserved == -1 ? "watch notifications" : "pings");
    if (n >= 0xFFFFFFFFull)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_stats: %llu records: must be below 2^32 - 1", (unsigned long long)n);
    sq.read = false;                                    /* from here on the arrays of the last read are overwritten */
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    int rc;
    for (Event &ev : sq.ev)
        if ((rc = ensure_event(ctx, ev)))
            return rc;
    const uint8_t *ds = bytes;
    if (!in_dev && len) {
        if ((rc = stage_in(ctx, sq.stream, bytes, len, s)))
            return rc;
        ds = (const uint8_t *)sq.stream.p;
    }
    const uint64_t nblk = (len + 15) / 16, tiles_s = (nblk + RP_TILE - 1) / RP_TILE;
    const size_t totals_bytes = align16(tiles_s * 4) + (tiles_s / SUPER + 1) * 8;
    const size_t n8 = n * 8 + 16, n4 = n * 4 + 16;
    if ((rc = ensure_dev(ctx, sq.word, nblk * 4 + 16)) || (rc = ensure_dev(ctx, sq.totals, totals_bytes)) ||
        (rc = ensure_dev(ctx, sq.tile_base, tiles_s * 8 + 16)) || (rc = ensure_dev(ctx, sq.fpos, n8)) ||
        (rc = ensure_dev(ctx, sq.err, n4)) || (rc = ensure_dev(ctx, sq.ver, n4)) || (rc = ensure_dev(ctx, sq.own, n8)) ||
        (rc = ensure_dev(ctx, sq.dlen, n4)) || (rc = ensure_dev(ctx, sq.mzxid, n8)) ||
        (rc = ensure_dev(ctx, sq.count, RQ_NCOUNTERS * 8)) || (rc = ensure_host(ctx, sq.h_count, RQ_NCOUNTERS * 8)))
        return rc;
    StatParams sp{};
    RepParams &p = sp.r;
    p.s = ds;
    p.len = len;
    p.xid_base = xb;
    p.n = n;
    p.word = (uint32_t *)sq.word.p;
    p.tile_total = (uint32_t *)sq.totals.p;
    p.super_total = (unsigned long long *)((uint8_t *)sq.totals.p + align16(tiles_s * 4));
    p.tile_base = (unsigned long long *)sq.tile_base.p;
    p.err = (int32_t *)sq.err.p;
    p.ver = (int32_t *)sq.ver.p;
    p.own = (long long *)sq.own.p;
    p.counters = (unsigned long long *)sq.count.p;
    sp.start = start;
    sp.fpos = (unsigned long long *)sq.fpos.p;
    sp.dlen = (int32_t *)sq.dlen.p;
    sp.mzxid = (long long *)sq.mzxid.p;
    unsigned long long *hc = (unsigned long long *)sq.h_count.p;
    CK(cudaMemsetAsync(p.counters, 0, RQ_NCOUNTERS * 8, s));
    CK(cudaMemsetAsync(p.counters + RQ_ERR, 0xFF, 8, s));
    CK(cudaMemsetAsync(p.tile_total, 0, totals_bytes, s));
    CK(cudaEventRecord(sq.ev[0], s));
    uint32_t launches = 0;
    /* 1. the frame chain from `start`, 2. the replies of the n records */
    RepParams pf = p;
    if (n && len) {
        if (opt_get(ctx, "stats_cand_shared", 0))
            regk_stats_cand_shared_kernel<<<(unsigned)tiles_s, RP_TILE, 0, s>>>(sp);
        else
            regk_stats_cand_kernel<<<(unsigned)tiles_s, RP_TILE, 0, s>>>(sp);
        CK(cudaGetLastError());
        launches++;
        uint32_t *J = nullptr;
        if ((rc = chain_pass(ctx, &pf, tiles_s, ~0ull, sq.cand, sq.mark, sq.jump, [&](const RepParams &q) {
                regk_children_seed_kernel<<<1, 256, 0, s>>>(q, nullptr, nullptr, 1, start);
            }, &J, &launches, who)))
            return rc;
        if (pf.C) {
            const uint64_t tiles_c = (pf.C + RP_TILE - 1) / RP_TILE;
            const size_t t2 = align16(tiles_c * 4) + (tiles_c / SUPER + 1) * 8;
            if ((rc = ensure_dev(ctx, sq.totals2, t2)))
                return rc;
            sp.r = pf;
            sp.r.tile_total = (uint32_t *)sq.totals2.p;
            sp.r.super_total = (unsigned long long *)((uint8_t *)sq.totals2.p + align16(tiles_c * 4));
            CK(cudaMemsetAsync(sq.totals2.p, 0, t2, s));
            regk_replies_chain_count_kernel<<<(unsigned)tiles_c, RP_TILE, 0, s>>>(sp.r);
            regk_stats_chain_kernel<<<(unsigned)tiles_c, RP_TILE, 0, s>>>(sp);
            CK(cudaGetLastError());
            launches += 3;
        }
    }
    CK(cudaEventRecord(sq.ev[1], s));
    CK(cudaMemcpyAsync(hc, p.counters, RQ_NCOUNTERS * 8, cudaMemcpyDeviceToHost, s));
    if ((rc = sync_or_fail(ctx, s, who)))
        return rc;
    /* refusals: a chain is read front to back, so the smallest failing reply is the first fault */
    if (hc[RQ_ERR] != ~0ull) {
        const uint64_t k = hc[RQ_ERR] >> 8;
        const uint32_t code = (uint32_t)(hc[RQ_ERR] & 0xFF);
        unsigned long long pos = 0;
        CK(cudaMemcpyAsync(&pos, sp.fpos + k, 8, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_stats: byte %llu: %s; expected the reply to record %llu (xid %d)",
            pos, stats_reason(code), (unsigned long long)k, (int32_t)((uint32_t)xb + (uint32_t)k));
    }
    if (hc[RQ_NREP] < n) {
        /* the chain stops before the n-th reply: the plausibility test where it stops names the reason */
        uint64_t stop = start;
        if (pf.C) {
            regk_replies_stop_kernel<<<(unsigned)((pf.C + 255) / 256), 256, 0, s>>>(pf);
            CK(cudaGetLastError());
            CK(cudaMemcpyAsync(hc + RQ_STOP, p.counters + RQ_STOP, 8, cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
            stop = std::max<uint64_t>(stop, hc[RQ_STOP]);
        }
        const uint64_t done = hc[RQ_NREP];
        uint8_t head[20] = {0};
        const uint64_t avail = len - stop, take = std::min<uint64_t>(avail, sizeof head);
        if (take) {
            CK(cudaMemcpyAsync(head, ds + stop, take, cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
        }
        StatHead h;
        const uint32_t code = stat_head(head, avail, xb, n, &h);   /* reads at most 20 bytes, all of them in head */
        const int32_t want = (int32_t)((uint32_t)xb + (uint32_t)done);
        if (code == ST_TRUNC)
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_stats: byte %llu: the stream ends before the reply to record %llu "
                                                   "(xid %d) is complete; %llu of %llu replies complete", (unsigned long long)stop,
                        (unsigned long long)done, want, (unsigned long long)done, (unsigned long long)n);
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_stats: byte %llu: %s (len %d, xid %d); expected the reply to record "
                                               "%llu (xid %d)", (unsigned long long)stop, code ? stats_reason(code) : "internal error",
                    h.len, h.xid, (unsigned long long)done, want);
    }
    float ms = 0;
    cudaEventElapsedTime(&ms, sq.ev[0], sq.ev[1]);
    const void *src[5] = {sq.err.p, sq.ver.p, sq.own.p, sq.dlen.p, sq.mzxid.p};
    if (!dev_out) {
        HostBuf *hb[5] = {&sq.h_err, &sq.h_ver, &sq.h_own, &sq.h_dlen, &sq.h_mzxid};
        const size_t sz[5] = {n * 4, n * 4, n * 8, n * 4, n * 8};
        for (int k = 0; k < 5; k++) {
            if ((rc = to_host(ctx, *hb[k], src[k], sz[k], s)))
                return rc;
            src[k] = hb[k]->p;
        }
        CK(cudaStreamSynchronize(s));
    }
    /* a subset framing's record list, kept with the read (the next regk_events_requests rewrites the framing's own) */
    sq.sub = ctx->ex_sub;
    sq.batch_n = ctx->last.n;
    if (sq.sub) {
        if ((rc = ensure_dev(ctx, sq.sub_rec, n * 8 + 16)))
            return rc;
        if (n)
            CK(cudaMemcpyAsync(sq.sub_rec.p, ctx->ex_rec, n * 8, cudaMemcpyDeviceToDevice, s));
        CK(cudaStreamSynchronize(s));
    }
    if ((rc = watch_read(ctx, false, (const int32_t *)sq.err.p, n, ctx->ex_sub ? ctx->ex_rec : nullptr, ctx->last.n)))
        return rc;
    sq.read = true;
    sq.gen = ctx->last.gen;
    sq.n = n;
    out->n = n;
    out->n_found = hc[RQ_FOUND];
    out->n_missing = hc[RQ_MISSING];
    out->n_error = hc[RQ_ERROR];
    out->n_skipped = hc[RQ_SKIP];
    out->consumed = n ? hc[RQ_CONSUMED] : start;
    out->flags = dev_out ? REGK_OUT_DEVICE : 0;
    out->launches = launches;
    out->err = (const int32_t *)src[0];
    out->version = (const int32_t *)src[1];
    out->ephemeral_owner = (const int64_t *)src[2];
    out->data_length = (const int32_t *)src[3];
    out->mzxid = (const int64_t *)src[4];
    out->kernel_ms = ms;
    return REGK_OK;
}

int regk_reconcile_stats(regk_ctx *ctx, const regk_stat_opts *o, uint32_t flags, regk_delta_owned *out)
{
    const char *who = "regk_reconcile_stats";
    if (!ctx || !o || !out)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_reconcile_stats: NULL argument");
    memset(out, 0, sizeof *out);
    ctx->rc.valid = false;
    ctx->rc.gen++;
    if (o->zk_flags > 1u)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_reconcile_stats: zk_flags %u is not 0 (persistent) or 1 (EPHEMERAL); a "
                                               "sequential or container mode makes a path key meaningless", o->zk_flags);
    if (o->zk_flags == 1u && o->session == 0)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_reconcile_stats: EPHEMERAL nodes need the session id they are sent on");
    const bool in_dev = flags & REGK_IN_DEVICE;
    if (o->known_mzxid && in_dev && ((uintptr_t)o->known_mzxid & 7u))
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_reconcile_stats: misaligned device known_mzxid (8-byte alignment needed)");
    if (ctx->pending)
        return fail(ctx, REGK_ERR_STATE, "regk_reconcile_stats: batches are still in flight; finish them first");
    regk_ctx::Stats &sq = ctx->sq;
    if (!sq.read)
        return fail(ctx, REGK_ERR_STATE, "regk_reconcile_stats: no stats on this context; call regk_read_stats first");
    if (sq.gen != ctx->last.gen || !ctx->last.path_off || !ctx->last.json_off || ctx->last.n != (sq.sub ? sq.batch_n : sq.n))
        return fail(ctx, REGK_ERR_STATE, "regk_reconcile_stats: a batch finished after regk_read_stats; its stats answer "
                                         "another batch's records");
    if (sq.sub && o->known_mzxid)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_reconcile_stats: known_mzxid with the stats of a regk_events_requests "
                                               "subset: the repair's own writes fire its watches and move mzxid");
    const uint64_t n = sq.sub ? sq.batch_n : sq.n;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    int rc;
    StatClassParams sp{};
    sp.err = (const int32_t *)sq.err.p;
    sp.own = (const long long *)sq.own.p;
    sp.dlen = (const int32_t *)sq.dlen.p;
    sp.mzxid = (const long long *)sq.mzxid.p;
    const int32_t *ver = (const int32_t *)sq.ver.p;
    uint32_t launches = 3;
    if (sq.sub) {
        /* the records whose watches did not fire read as SAME: a node the batch owns at its payload length */
        EvStatFill f{};
        f.n = n;
        f.m = sq.n;
        f.json_off = ctx->last.json_off;
        f.want = o->zk_flags == 1u ? (long long)o->session : 0ll;
        f.rec = (const unsigned long long *)sq.sub_rec.p;
        f.s_err = sp.err;
        f.s_ver = ver;
        f.s_dlen = sp.dlen;
        f.s_own = sp.own;
        if ((rc = ensure_dev(ctx, sq.f_err, n * 4 + 16)) || (rc = ensure_dev(ctx, sq.f_ver, n * 4 + 16)) ||
            (rc = ensure_dev(ctx, sq.f_own, n * 8 + 16)) || (rc = ensure_dev(ctx, sq.f_dlen, n * 4 + 16)))
            return rc;
        f.err = (int32_t *)sq.f_err.p;
        f.ver = (int32_t *)sq.f_ver.p;
        f.own = (long long *)sq.f_own.p;
        f.dlen = (int32_t *)sq.f_dlen.p;
        if (n)
            regk_events_stat_fill_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(f);
        if (f.m)
            regk_events_stat_scatter_kernel<<<(unsigned)((f.m + 255) / 256), 256, 0, s>>>(f);
        CK(cudaGetLastError());
        launches += (n ? 1 : 0) + (f.m ? 1 : 0);
        sp.err = f.err;
        sp.own = f.own;
        sp.dlen = f.dlen;
        sp.mzxid = nullptr;                         /* read only against known_mzxid */
        ver = f.ver;
    }
    sp.known_mzxid = (const long long *)o->known_mzxid;
    if (o->known_mzxid && !in_dev) {
        if ((rc = stage_in(ctx, sq.known, o->known_mzxid, n * 8, s)))
            return rc;
        sp.known_mzxid = (const long long *)sq.known.p;
    }
    /* no observed side: m = 0; the compact pass takes each update / replace entry's version from the stats, through
       match[i] = the record itself */
    ReconcileParams &p = sp.rc;
    p.o_version = ver;
    p.want = o->zk_flags == 1u ? (long long)o->session : 0ll;
    if ((rc = reconcile_prepare(ctx, n, 0, true, &p)))
        return rc;
    regk_stats_class_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(sp);
    regk_stats_mark_kernel<<<p.tiles_r, RC_TILE, 0, s>>>(sp);
    regk_reconcile_compact_kernel<<<p.tiles_r, RC_TILE, 0, s>>>(p);
    CK(cudaGetLastError());
    unsigned long long *hc = (unsigned long long *)ctx->rc.h_count.p;
    CK(cudaMemcpyAsync(hc, p.counters, RC_NCOUNTERS * 8, cudaMemcpyDeviceToHost, s));
    if ((rc = sync_or_fail(ctx, s, who)))
        return rc;
    if (hc[RC_C_BAD] != ~0ull) {
        int32_t e = 0;
        CK(cudaMemcpy(&e, sp.err + hc[RC_C_BAD], 4, cudaMemcpyDeviceToHost));
        return fail(ctx, REGK_ERR_STATE, "regk_reconcile_stats: record %llu's reply carries error %d: the state of its node is "
                                         "unknown, and no repair over it is right", hc[RC_C_BAD], e);
    }
    rc = reconcile_finish(ctx, p, hc, true, o->zk_flags, flags, launches, &out->d, &out->replace, &out->n_replace, who);
    out->d.obs_cls = nullptr;
    return rc;
}

static const char *events_reason(uint32_t code)
{
    switch (code) {
    case EV_TRUNC: return "the stream ends inside the frame";
    case EV_BAD_LEN: return "a frame length below 16 (no room for a ReplyHeader)";
    case EV_NEG_XID: return "a negative xid other than -1 (notification) or -2 (ping), outside the reply range";
    case EV_XID_RANGE: return "an xid outside the reply range";
    case EV_NOTE_LEN: return "a notification whose length is not 28 + its path length";
    case EV_NEG_PATH: return "a notification with a negative path length";
    case EV_NOTE_ERR: return "a notification with err != 0";
    case EV_TYPE: return "a notification whose type is outside -1 .. 7";
    case EV_PING_BODY: return "a ping with a body";
    case EV_SW_BODY: return "a SetWatches reply (xid -8) with a body";
    case EV_SW_ERR: return "a SetWatches reply (xid -8) with err != 0";
    default: return "internal error";
    }
}

/* The tables regk_read_events maps paths with, for the batch finished last: the record table, the directory set and
   its table, zeroed marks and pending counts.  Once per batch generation. */
static int events_build(regk_ctx *ctx, const char *who)
{
    regk_ctx::Events &ev = ctx->evq;
    cudaStream_t s = ctx->stream;
    const uint64_t n = ctx->last.n;
    int rc;
    ev.built = ev.read = false;
    ev.d = ev.prefixes = ev.n_unlisted = 0;
    if (n && !ctx->last.alias && (rc = children_dirs(ctx, ev, false)))
        return rc;
    const uint64_t d = ev.d;
    uint64_t sr = 1024, sd = 1024;
    while (sr < 2 * n)
        sr <<= 1;
    while (sd < 2 * d)
        sd <<= 1;
    if (sr > (1ull << 32))
        return fail(ctx, REGK_ERR_INVALID_ARG, "%s: %llu records are too many for one table", who, (unsigned long long)n);
    if ((rc = ensure_dev(ctx, ev.zero, n * 4 + 16)) || (rc = ensure_dev(ctx, ev.slot, n * 4 + 16)) ||
        (rc = ensure_dev(ctx, ev.t_rec, sr * 4)) || (rc = ensure_dev(ctx, ev.t_dir, sd * 4)) ||
        (rc = ensure_dev(ctx, ev.rec_mark, n * 4 + 16)) || (rc = ensure_dev(ctx, ev.dir_mark, d * 4 + 16)) ||
        (rc = ensure_dev(ctx, ev.dirty, 16)))
        return rc;
    CK(cudaMemsetAsync(ev.zero.p, 0, n * 4 + 16, s));
    CK(cudaMemsetAsync(ev.t_rec.p, 0, sr * 4, s));
    CK(cudaMemsetAsync(ev.t_dir.p, 0, sd * 4, s));
    CK(cudaMemsetAsync(ev.rec_mark.p, 0, n * 4 + 16, s));
    CK(cudaMemsetAsync(ev.dir_mark.p, 0, d * 4 + 16, s));
    CK(cudaMemsetAsync(ev.dirty.p, 0, 16, s));
    if (n) {
        /* every record "found": the first record with a path keeps its slot */
        RepParams rp{};
        rp.n = n;
        rp.err = (int32_t *)ev.zero.p;
        rp.d_path = ctx->last.path_bytes;
        rp.d_path_off = ctx->last.path_off;
        rp.table = (uint32_t *)ev.t_rec.p;
        rp.mask_t = (uint32_t)(sr - 1);
        rp.slot = (uint32_t *)ev.slot.p;
        regk_replies_insert_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(rp);
    }
    if (d) {
        EvDirParams dp{};
        dp.d_path = ctx->last.path_bytes;
        dp.d_path_off = ctx->last.path_off;
        dp.dir_rec = (const unsigned long long *)ev.drec.p;
        dp.dir_len = (const uint32_t *)ev.dlen.p;
        dp.d = d;
        dp.table = (uint32_t *)ev.t_dir.p;
        dp.mask = (uint32_t)(sd - 1);
        regk_events_dir_insert_kernel<<<(unsigned)((d + 255) / 256), 256, 0, s>>>(dp);
    }
    CK(cudaGetLastError());
    if ((rc = sync_or_fail(ctx, s, who)))
        return rc;
    ev.mask_r = (uint32_t)(sr - 1);
    ev.mask_d = (uint32_t)(sd - 1);
    ev.rec_epoch = ev.dir_epoch = 1;
    ev.n = n;
    ev.gen = ctx->last.gen;
    ev.built = true;
    return REGK_OK;
}

int regk_read_events(regk_ctx *ctx, const uint8_t *bytes, uint64_t len, uint64_t start, const regk_events_opts *o,
    regk_events *out)
{
    const char *who = "regk_read_events";
    if (!ctx || !o || !out)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_events: NULL argument");
    memset(out, 0, sizeof *out);
    regk_ctx::Events &ev = ctx->evq;
    if (ctx->pending)
        return fail(ctx, REGK_ERR_STATE, "regk_read_events: batches are still in flight; finish them first");
    if (!ctx->last.path_off || !ctx->last.path_bytes)
        return fail(ctx, REGK_ERR_STATE, "regk_read_events: no finished batch with a path stream on this context: events "
                                         "map to the records of the batch finished last");
    if (ctx->last.n >= 0xFFFFFFFEull)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_events: batch too large");
    if (!bytes && len)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_events: NULL stream of %llu bytes", (unsigned long long)len);
    if (start > len)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_events: start %llu is past the stream's %llu bytes",
            (unsigned long long)start, (unsigned long long)len);
    const bool in_dev = o->flags & REGK_IN_DEVICE, dev_out = o->flags & REGK_OUT_DEVICE;
    if (in_dev && ((uintptr_t)bytes & 15u))
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_events: misaligned device stream (16-byte alignment needed)");
    const int32_t xb = o->xid_base;
    const uint64_t nx = o->n_xids;
    for (int32_t reserved : {-1, -2})
        if ((uint64_t)((uint32_t)reserved - (uint32_t)xb) < nx)
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_events: the reply xids [%d, %d + %llu) cover %d, which ZooKeeper "
                                                   "uses for %s", xb, xb, (unsigned long long)nx, reserved,
                        reserved == -1 ? "watch notifications" : "pings");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    int rc;
    if (!ev.built || ev.gen != ctx->last.gen) {
        if ((rc = events_build(ctx, who)))
            return rc;
    }
    for (Event &e : ev.ev)
        if ((rc = ensure_event(ctx, e)))
            return rc;
    regk_ctx::Watch &wq = watch_state(ctx);
    const bool sw = wq.gate;                    /* SetWatches replies are frames of the stream */
    if ((rc = ensure_dev(ctx, wq.zmax, 16)))
        return rc;
    const uint8_t *ds = bytes;
    if (!in_dev && len) {
        if ((rc = stage_in(ctx, ev.stream, bytes, len, s)))
            return rc;
        ds = (const uint8_t *)ev.stream.p;
    }
    const uint64_t nblk = (len + 15) / 16, tiles_s = (nblk + RP_TILE - 1) / RP_TILE;
    const size_t totals_bytes = align16(tiles_s * 4) + (tiles_s / SUPER + 1) * 8;
    if ((rc = ensure_dev(ctx, ev.word, nblk * 4 + 16)) || (rc = ensure_dev(ctx, ev.ftotals, totals_bytes)) ||
        (rc = ensure_dev(ctx, ev.tile_base, tiles_s * 8 + 16)) || (rc = ensure_dev(ctx, ev.ecount, EQ_NCOUNTERS * 8)) ||
        (rc = ensure_host(ctx, ev.h_ecount, EQ_NCOUNTERS * 8 + 16)))
        return rc;
    EvParams ep{};
    RepParams &p = ep.r;
    p.s = ds;
    p.len = len;
    p.xid_base = xb;
    p.n = nx;
    p.word = (uint32_t *)ev.word.p;
    p.tile_total = (uint32_t *)ev.ftotals.p;
    p.super_total = (unsigned long long *)((uint8_t *)ev.ftotals.p + align16(tiles_s * 4));
    p.tile_base = (unsigned long long *)ev.tile_base.p;
    p.counters = (unsigned long long *)ev.ecount.p;
    ep.start = start;
    ep.d_path = ctx->last.path_bytes;
    ep.d_path_off = ctx->last.path_off;
    ep.t_rec = (const uint32_t *)ev.t_rec.p;
    ep.mask_r = ev.mask_r;
    ep.t_dir = (const uint32_t *)ev.t_dir.p;
    ep.mask_d = ev.mask_d;
    ep.dir_rec = (const unsigned long long *)ev.drec.p;
    ep.dir_len = (const uint32_t *)ev.dlen.p;
    ep.rec_mark = (uint32_t *)ev.rec_mark.p;
    ep.dir_mark = (uint32_t *)ev.dir_mark.p;
    ep.rec_epoch = ev.rec_epoch;
    ep.dir_epoch = ev.dir_epoch;
    ep.dirty = (unsigned long long *)ev.dirty.p;
    unsigned long long *hc = (unsigned long long *)ev.h_ecount.p;
    CK(cudaMemsetAsync(p.counters, 0, EQ_NCOUNTERS * 8, s));
    CK(cudaMemsetAsync(p.tile_total, 0, totals_bytes, s));
    CK(cudaEventRecord(ev.ev[0], s));
    uint32_t launches = 0;
    /* 1. the frame chain from `start` and where it stops */
    RepParams pf = p;
    if (len > start) {
        if (sw)
            regk_events_sw_cand_kernel<<<(unsigned)tiles_s, RP_TILE, 0, s>>>(ep);
        else
            regk_events_cand_kernel<<<(unsigned)tiles_s, RP_TILE, 0, s>>>(ep);
        CK(cudaGetLastError());
        launches++;
        uint32_t *J = nullptr;
        if ((rc = chain_pass(ctx, &pf, tiles_s, ~0ull, ev.cand, ev.mark, ev.jump, [&](const RepParams &q) {
                regk_children_seed_kernel<<<1, 256, 0, s>>>(q, nullptr, nullptr, 1, start);
            }, &J, &launches, who)))
            return rc;
        if (pf.C) {
            regk_replies_stop_kernel<<<(unsigned)((pf.C + 255) / 256), 256, 0, s>>>(pf);
            CK(cudaGetLastError());
            launches++;
        }
    }
    CK(cudaMemcpyAsync(hc, p.counters, EQ_NCOUNTERS * 8, cudaMemcpyDeviceToHost, s));
    if ((rc = sync_or_fail(ctx, s, who)))
        return rc;
    const uint64_t stop = std::max<uint64_t>(start, hc[RQ_STOP]);
    bool partial = false;
    if (stop < len) {
        /* the first position the chain does not pass: a frame still arriving, or a fault.  Nothing has been marked. */
        uint8_t head[32] = {0};
        const uint64_t avail = len - stop, take = std::min<uint64_t>(avail, sizeof head);
        CK(cudaMemcpyAsync(head, ds + stop, take, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        EvHead h;
        /* reads at most 32 bytes, all of them in head */
        const uint32_t code = sw ? ev_sw_head(head, avail, xb, nx, &h) : ev_head(head, avail, xb, nx, &h);
        if (code != EV_TRUNC)
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_events: byte %llu: %s (len %d, xid %d)", (unsigned long long)stop,
                code ? events_reason(code) : "internal error", h.len, h.xid);
        partial = true;
    }
    /* 2. the events of the chain, mapped and marked */
    const uint64_t C = pf.C;
    if ((rc = ensure_dev(ctx, ev.pos, C * 8 + 16)) || (rc = ensure_dev(ctx, ev.subject, C * 8 + 16)) ||
        (rc = ensure_dev(ctx, ev.zxid, C * 8 + 16)) || (rc = ensure_dev(ctx, ev.type, C * 4 + 16)) ||
        (rc = ensure_dev(ctx, ev.state, C * 4 + 16)) || (rc = ensure_dev(ctx, ev.kind, C + 16)))
        return rc;
    ep.r = pf;
    ep.pos = (unsigned long long *)ev.pos.p;
    ep.subject = (unsigned long long *)ev.subject.p;
    ep.zxid = (long long *)ev.zxid.p;
    ep.type = (int32_t *)ev.type.p;
    ep.state = (int32_t *)ev.state.p;
    ep.kind = (uint8_t *)ev.kind.p;
    if (C) {
        const uint64_t tiles_c = (C + RP_TILE - 1) / RP_TILE;
        const size_t t2 = align16(tiles_c * 4) + (tiles_c / SUPER + 1) * 8;
        if ((rc = ensure_dev(ctx, ev.ntotals, t2)))
            return rc;
        ep.tile_total = (uint32_t *)ev.ntotals.p;
        ep.super_total = (unsigned long long *)((uint8_t *)ev.ntotals.p + align16(tiles_c * 4));
        CK(cudaMemsetAsync(ev.ntotals.p, 0, t2, s));
        CK(cudaMemsetAsync(wq.zmax.p, 0, 8, s));
        regk_events_count_kernel<<<(unsigned)tiles_c, RP_TILE, 0, s>>>(ep);
        regk_events_kernel<<<(unsigned)tiles_c, RP_TILE, 0, s>>>(ep);
        regk_events_zxid_kernel<<<(unsigned)((C + 255) / 256), 256, 0, s>>>(pf, (long long *)wq.zmax.p);
        CK(cudaGetLastError());
        launches += 3;
    }
    CK(cudaEventRecord(ev.ev[1], s));
    CK(cudaMemcpyAsync(hc, p.counters, EQ_NCOUNTERS * 8, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(hc + EQ_NCOUNTERS, ev.dirty.p, 16, cudaMemcpyDeviceToHost, s));
    long long zmax = 0;
    if (C)
        CK(cudaMemcpyAsync(&zmax, wq.zmax.p, 8, cudaMemcpyDeviceToHost, s));
    if ((rc = sync_or_fail(ctx, s, who)))
        return rc;
    const uint64_t ne = C ? hc[EQ_NEV] : 0;
    float ms = 0;
    cudaEventElapsedTime(&ms, ev.ev[0], ev.ev[1]);
    const void *src[6] = {ev.pos.p, ev.type.p, ev.state.p, ev.zxid.p, ev.kind.p, ev.subject.p};
    if (!dev_out) {
        HostBuf *hb[6] = {&ev.h_pos, &ev.h_type, &ev.h_state, &ev.h_zxid, &ev.h_kind, &ev.h_subject};
        const size_t sz[6] = {ne * 8, ne * 4, ne * 4, ne * 8, ne, ne * 8};
        for (int k = 0; k < 6; k++) {
            if ((rc = to_host(ctx, *hb[k], src[k], sz[k], s)))
                return rc;
            src[k] = hb[k]->p;
        }
        CK(cudaStreamSynchronize(s));
    }
    ev.read = true;
    wq.zxid = std::max(wq.zxid, zmax);
    out->n_events = ne;
    out->n_pings = hc[EQ_PING];
    out->n_replies = hc[EQ_REPLY];
    out->n_unmatched = hc[EQ_UNMATCHED];
    out->n_other = hc[EQ_OTHER];
    out->consumed = stop;
    out->n_dirty_recs = hc[EQ_NCOUNTERS];
    out->n_dirty_dirs = hc[EQ_NCOUNTERS + 1];
    out->partial = partial ? 1u : 0u;
    out->flags = dev_out ? REGK_OUT_DEVICE : 0;
    out->launches = launches;
    out->pos = (const uint64_t *)src[0];
    out->type = (const int32_t *)src[1];
    out->state = (const int32_t *)src[2];
    out->zxid = (const int64_t *)src[3];
    out->subject_kind = (const uint8_t *)src[4];
    out->subject = (const uint64_t *)src[5];
    out->kernel_ms = ms;
    return REGK_OK;
}

/* The pending records (dirs == false) or directories of the current epoch, ascending, into evq.item / prec / plen[dirs];
   *m = their number. */
static int events_pending(regk_ctx *ctx, bool dirs, uint64_t *m, uint32_t *launches, const char *who)
{
    regk_ctx::Events &ev = ctx->evq;
    cudaStream_t s = ctx->stream;
    const int w = dirs ? 1 : 0;
    const uint64_t N = dirs ? ev.d : ev.n;
    const uint64_t tiles = (N + RP_TILE - 1) / RP_TILE;
    const size_t tb = align16(tiles * 4) + (tiles / SUPER + 1) * 8;
    int rc;
    if ((rc = ensure_dev(ctx, ev.ptotals, tb + 16)) || (rc = ensure_dev(ctx, ev.pcount, 16)) ||
        (rc = ensure_dev(ctx, ev.item[w], N * 8 + 16)) || (rc = ensure_dev(ctx, ev.prec[w], N * 8 + 16)) ||
        (rc = ensure_dev(ctx, ev.plen[w], N * 4 + 16)))
        return rc;
    *m = 0;
    if (!N)
        return REGK_OK;
    EvPendParams pp{};
    pp.n = N;
    pp.mark = (const uint32_t *)(dirs ? ev.dir_mark.p : ev.rec_mark.p);
    pp.shift = dirs ? 0u : 3u;
    pp.epoch = dirs ? ev.dir_epoch : ev.rec_epoch;
    pp.path_off = ctx->last.path_off;
    pp.dir_rec = dirs ? (const unsigned long long *)ev.drec.p : nullptr;
    pp.dir_len = dirs ? (const uint32_t *)ev.dlen.p : nullptr;
    pp.tile_total = (uint32_t *)ev.ptotals.p;
    pp.super_total = (unsigned long long *)((uint8_t *)ev.ptotals.p + align16(tiles * 4));
    pp.item = (unsigned long long *)ev.item[w].p;
    pp.rec = (unsigned long long *)ev.prec[w].p;
    pp.len = (uint32_t *)ev.plen[w].p;
    pp.count = (unsigned long long *)ev.pcount.p;
    CK(cudaMemsetAsync(ev.ptotals.p, 0, tb, s));
    regk_events_pending_count_kernel<<<(unsigned)tiles, RP_TILE, 0, s>>>(pp);
    regk_events_pending_kernel<<<(unsigned)tiles, RP_TILE, 0, s>>>(pp);
    CK(cudaGetLastError());
    *launches += 2;
    unsigned long long cnt = 0;
    CK(cudaMemcpyAsync(&cnt, pp.count, 8, cudaMemcpyDeviceToHost, s));
    if ((rc = sync_or_fail(ctx, s, who)))
        return rc;
    *m = cnt;
    return REGK_OK;
}

int regk_events_requests(regk_ctx *ctx, const regk_jute_opts *o, regk_frames *out)
{
    const char *who = "regk_events_requests";
    if (!ctx || !o || !out)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_events_requests: NULL argument");
    memset(out, 0, sizeof *out);
    const bool exists = o->op == REGK_ZK_EXISTS;
    if (!exists && o->op != REGK_ZK_GETCHILDREN)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_events_requests: op %u is not exists (3) or getChildren (8)", o->op);
    if (o->group != 0)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_events_requests: reads cannot go in a multi transaction (group %u)", o->group);
    if (ctx->pending)
        return fail(ctx, REGK_ERR_STATE, "regk_events_requests: batches are still in flight; finish them first");
    regk_ctx::Events &ev = ctx->evq;
    if (!ev.read || ev.gen != ctx->last.gen || !ctx->last.path_off)
        return fail(ctx, REGK_ERR_STATE, "regk_events_requests: no regk_read_events call for the batch finished last");
    if (exists && (!ctx->last.json_off || ctx->last.n != ctx->last.json_n))
        return fail(ctx, REGK_ERR_STATE, "regk_events_requests: no finished batch with both a path and a payload stream on "
                                         "this context: the exists replies are classed against the payload lengths");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    int rc;
    uint64_t m = 0, total = 0;
    uint32_t launches = 0;
    const int w = exists ? 0 : 1;
    if ((rc = watch_forget_unread(ctx, !exists, nullptr)))
        return rc;
    if ((rc = events_pending(ctx, !exists, &m, &launches, who)))
        return rc;
    regk_jute_opts oo = *o;
    oo.flags = (o->flags & REGK_OUT_DEVICE) | REGK_ZK_WATCH;    /* watches are one-shot: every re-check re-arms */
    FrameSrc src{};
    src.who = who;
    if (exists) {
        ctx->ex_valid = false;
        if ((rc = pack_strings(ctx, m, ctx->last.path_bytes, ctx->last.path_off, (const unsigned long long *)ev.prec[w].p,
                 (const uint32_t *)ev.plen[w].p, ev.ptotals, ev.pbytes, ev.poff, &total, &launches)))
            return rc;
        src = FrameSrc{m, (const uint8_t *)ev.pbytes.p, (const unsigned long long *)ev.poff.p, nullptr, nullptr, who};
        if ((rc = frame_requests(ctx, src, &oo, ev.frames, out)))
            return rc;
        ctx->ex_valid = true;
        ctx->ex_gen = ctx->last.gen;
        ctx->ex_xid = o->xid_base;
        ctx->ex_n = m;
        ctx->ex_sub = true;
        ctx->ex_rec = (const unsigned long long *)ev.item[w].p;
        ev.rec_epoch++;
        if ((rc = watch_framed(ctx, false, true)))
            return rc;
    } else {
        regk_ctx::Children &ch = ctx->ch;
        ch.framed = false;
        if ((rc = ensure_dev(ctx, ch.drec, m * 8 + 8)) || (rc = ensure_dev(ctx, ch.dlen, m * 4 + 8)) ||
            (rc = ensure_dev(ctx, ch.unlisted, 8)))
            return rc;
        if (m) {
            CK(cudaMemcpyAsync(ch.drec.p, ev.prec[w].p, m * 8, cudaMemcpyDeviceToDevice, s));
            CK(cudaMemcpyAsync(ch.dlen.p, ev.plen[w].p, m * 4, cudaMemcpyDeviceToDevice, s));
        }
        if ((rc = pack_strings(ctx, m, ctx->last.path_bytes, ctx->last.path_off, (const unsigned long long *)ch.drec.p,
                 (const uint32_t *)ch.dlen.p, ch.totals, ch.dbytes, ch.doff, &total, &launches)))
            return rc;
        src = FrameSrc{m, (const uint8_t *)ch.dbytes.p, (const unsigned long long *)ch.doff.p, nullptr, nullptr, who};
        if ((rc = frame_requests(ctx, src, &oo, ch.frames[0], out)))
            return rc;
        ch.framed = true;
        ch.gen = ctx->last.gen;
        ch.n = ctx->last.n;
        ch.d = m;
        ch.n_unlisted = 0;
        ch.prefixes = ev.prefixes;
        ch.xid = o->xid_base;
        ch.keep_drec = (const unsigned long long *)ev.drec.p;
        ch.keep_dlen = (const uint32_t *)ev.dlen.p;
        ch.keep_d = ev.d;
        ch.sub_item = (const unsigned long long *)ev.item[w].p;
        ev.dir_epoch++;
        if ((rc = watch_framed(ctx, true, true)))
            return rc;
    }
    CK(cudaMemsetAsync((unsigned long long *)ev.dirty.p + w, 0, 8, s));
    CK(cudaStreamSynchronize(s));
    out->launches += launches;
    return REGK_OK;
}

int regk_setwatches_requests(regk_ctx *ctx, const regk_setwatches_opts *o, regk_setwatches *out)
{
    const char *who = "regk_setwatches_requests";
    if (!ctx || !o || !out)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_setwatches_requests: NULL argument");
    memset(out, 0, sizeof *out);
    if (o->flags & ~(uint32_t)REGK_OUT_DEVICE)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_setwatches_requests: unknown flag bits 0x%x (only REGK_OUT_DEVICE)",
            o->flags & ~(uint32_t)REGK_OUT_DEVICE);
    if (o->max_frame >= 0x80000000u)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_setwatches_requests: max_frame %u is 2^31 or more; a frame's length is "
                                               "a signed 32-bit int", o->max_frame);
    if (ctx->pending)
        return fail(ctx, REGK_ERR_STATE, "regk_setwatches_requests: batches are still in flight; finish them first");
    if (!ctx->last.path_off || !ctx->last.path_bytes)
        return fail(ctx, REGK_ERR_STATE, "regk_setwatches_requests: no finished batch with a path stream on this context: the "
                                         "watches are the ones its reads armed");
    if (ctx->last.n >= 0xFFFFFFFEull)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_setwatches_requests: batch too large");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    regk_ctx::Events &ev = ctx->evq;
    int rc;
    if (!ev.built || ev.gen != ctx->last.gen) {
        if ((rc = events_build(ctx, who)))
            return rc;
    }
    regk_ctx::Watch &w = watch_state(ctx);
    for (Event &e : w.ev)
        if ((rc = ensure_event(ctx, e)))
            return rc;
    const uint64_t n = ctx->last.n, d = ev.d;
    uint32_t launches = 0;
    /* 1. the split's bound: the longest path, once per batch generation */
    if (!w.lmax_ok) {
        if ((rc = ensure_dev(ctx, w.lmax_d, 16)))
            return rc;
        CK(cudaMemsetAsync(w.lmax_d.p, 0, 4, s));
        if (n) {
            regk_sw_lmax_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(ctx->last.path_off, n, (uint32_t *)w.lmax_d.p);
            CK(cudaGetLastError());
            launches++;
        }
        uint32_t lm = 0;
        CK(cudaMemcpyAsync(&lm, w.lmax_d.p, 4, cudaMemcpyDeviceToHost, s));
        if ((rc = sync_or_fail(ctx, s, who)))
            return rc;
        w.lmax = lm;
        w.lmax_ok = true;
    }
    const uint64_t Lmax = 4ull + w.lmax, mf = o->max_frame ? o->max_frame : 131072u;
    if (mf < SW_OVERHEAD + 2 * Lmax)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_setwatches_requests: max_frame %llu is below this batch's minimum of %llu "
                                               "(32 + 2 x (4 + its longest path, %u bytes))", (unsigned long long)mf,
                    (unsigned long long)(SW_OVERHEAD + 2 * Lmax), w.lmax);
    const uint64_t B = mf - SW_OVERHEAD - Lmax;
    /* 2. what is in flight counts as NONE */
    uint8_t *rk = nullptr, *dk = nullptr;
    if ((rc = watch_kinds(ctx, false, n, &rk)) || (rc = watch_kinds(ctx, true, d, &dk)))
        return rc;
    if ((rc = watch_forget_unread(ctx, false, &launches)) || (rc = watch_forget_unread(ctx, true, &launches)))
        return rc;
    /* 3. classify: the lists, the re-pend marks, per-tile counts and bytes */
    const uint64_t tiles_r = (n + RP_TILE - 1) / RP_TILE, tiles_d = (d + RP_TILE - 1) / RP_TILE;
    const size_t reg_r = align16(tiles_r * 4) + (tiles_r / SUPER + 1) * 8, reg_d = align16(tiles_d * 4) + (tiles_d / SUPER + 1) * 8;
    const size_t totals_bytes = 4 * reg_r + 2 * reg_d;
    if ((rc = ensure_dev(ctx, w.totals, totals_bytes)) || (rc = ensure_dev(ctx, w.count, SWQ_N * 8 + 16)) ||
        (rc = ensure_dev(ctx, w.cls, n + d + 16)))
        return rc;
    SwParams sp{};
    sp.n = n;
    sp.d = d;
    sp.tiles_r = (uint32_t)tiles_r;
    sp.path_off = ctx->last.path_off;
    sp.slot = (const uint32_t *)ev.slot.p;
    sp.t_rec = (const uint32_t *)ev.t_rec.p;
    sp.dir_rec = (const unsigned long long *)ev.drec.p;
    sp.dir_len = (const uint32_t *)ev.dlen.p;
    sp.rec_kind = rk;
    sp.dir_kind = dk;
    sp.rec_mark = (uint32_t *)ev.rec_mark.p;
    sp.dir_mark = (uint32_t *)ev.dir_mark.p;
    sp.rec_epoch = ev.rec_epoch;
    sp.dir_epoch = ev.dir_epoch;
    sp.dirty = (unsigned long long *)ev.dirty.p;
    sp.counters = (unsigned long long *)w.count.p;
    sp.cls = (uint8_t *)w.cls.p;
    {
        uint8_t *t = (uint8_t *)w.totals.p;
        for (int k = 0; k < SWT_N; k++) {
            const bool dr = k >= SWT_CC;
            const uint64_t tiles = dr ? tiles_d : tiles_r;
            sp.tt[k] = (uint32_t *)t;
            sp.st[k] = (unsigned long long *)(t + align16(tiles * 4));
            t += dr ? reg_d : reg_r;
        }
    }
    CK(cudaMemsetAsync(w.totals.p, 0, totals_bytes, s));
    CK(cudaMemsetAsync(w.count.p, 0, SWQ_N * 8, s));
    CK(cudaEventRecord(w.ev[0], s));
    const unsigned grid = (unsigned)(tiles_r + tiles_d);
    if (grid) {
        regk_sw_classify_kernel<<<grid, RP_TILE, 0, s>>>(sp);
        CK(cudaGetLastError());
        launches++;
    }
    uint64_t sums[SWT_N] = {};
    std::vector<unsigned long long> sup(4 * (tiles_r / SUPER + 1) + 2 * (tiles_d / SUPER + 1));
    for (int k = 0, at = 0; k < SWT_N; k++) {
        const uint64_t ns = (k >= SWT_CC ? tiles_d : tiles_r) / SUPER + 1;
        CK(cudaMemcpyAsync(sup.data() + at, sp.st[k], ns * 8, cudaMemcpyDeviceToHost, s));
        at += (int)ns;
    }
    unsigned long long hq[SWQ_N + 2] = {};
    CK(cudaMemcpyAsync(hq, w.count.p, SWQ_N * 8, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(hq + SWQ_N, ev.dirty.p, 16, cudaMemcpyDeviceToHost, s));
    if ((rc = sync_or_fail(ctx, s, who)))
        return rc;
    for (int k = 0, at = 0; k < SWT_N; k++) {
        const uint64_t ns = (k >= SWT_CC ? tiles_d : tiles_r) / SUPER + 1;
        for (uint64_t q = 0; q < ns; q++)
            sums[k] += sup[at + q];
        at += (int)ns;
    }
    const uint64_t nD = sums[SWT_DC], nE = sums[SWT_EC], nC = sums[SWT_CC], m = nD + nE + nC;
    const uint64_t total_s = sums[SWT_DB] + sums[SWT_EB] + sums[SWT_CB];
    /* 4. place: entry j's path, length and prefix s_j */
    if ((rc = ensure_dev(ctx, w.ent_src, m * 8 + 16)) || (rc = ensure_dev(ctx, w.ent_s, m * 8 + 16)) ||
        (rc = ensure_dev(ctx, w.ent_len, m * 4 + 16)))
        return rc;
    sp.nD = nD;
    sp.nE = nE;
    sp.m = m;
    sp.bD = sums[SWT_DB];
    sp.bE = sums[SWT_EB];
    sp.total_s = total_s;
    sp.B = B;
    sp.zxid = w.zxid;
    sp.ent_src = (unsigned long long *)w.ent_src.p;
    sp.ent_s = (unsigned long long *)w.ent_s.p;
    sp.ent_len = (uint32_t *)w.ent_len.p;
    sp.path_bytes = ctx->last.path_bytes;
    uint64_t F = 0;
    if (m) {
        regk_sw_place_kernel<<<grid, RP_TILE, 0, s>>>(sp);
        CK(cudaGetLastError());
        launches++;
        unsigned long long last_s = 0;
        CK(cudaMemcpyAsync(&last_s, sp.ent_s + (m - 1), 8, cudaMemcpyDeviceToHost, s));
        if ((rc = sync_or_fail(ctx, s, who)))
            return rc;
        F = last_s / B + 1;
    }
    /* 5. the frames: entries, then headers and count words over the bytes between them */
    const uint64_t total = SW_OVERHEAD * F + total_s;
    FrameBufs &fb = w.frames;
    if ((rc = ensure_dev(ctx, fb.bytes, total + 16)) || (rc = ensure_dev(ctx, fb.off, (F + 1) * 8)))
        return rc;
    sp.out = (uint8_t *)fb.bytes.p;
    sp.frame_off = (unsigned long long *)fb.off.p;
    sp.F = F;
    if (m) {
        regk_sw_write_kernel<<<(unsigned)((m + RP_TILE - 1) / RP_TILE), RP_TILE, 0, s>>>(sp);
        regk_sw_head_kernel<<<(unsigned)((F + 255) / 256), 256, 0, s>>>(sp);
        CK(cudaGetLastError());
        launches += 2;
    } else {
        CK(cudaMemsetAsync(fb.off.p, 0, 8, s));
    }
    CK(cudaEventRecord(w.ev[1], s));
    if ((rc = sync_or_fail(ctx, s, who)))
        return rc;
    float ms = 0;
    cudaEventElapsedTime(&ms, w.ev[0], w.ev[1]);
    const bool dev_out = o->flags & REGK_OUT_DEVICE;
    const void *src[2] = {fb.bytes.p, fb.off.p};
    if (!dev_out) {
        if ((rc = to_host(ctx, fb.h_bytes, fb.bytes.p, total, s)) || (rc = to_host(ctx, fb.h_off, fb.off.p, (F + 1) * 8, s)))
            return rc;
        CK(cudaStreamSynchronize(s));
        src[0] = fb.h_bytes.p;
        src[1] = fb.h_off.p;
    }
    w.gate = true;
    out->n_data = nD;
    out->n_exist = nE;
    out->n_child = nC;
    out->n_repend_recs = hq[SWQ_REPEND_R];
    out->n_repend_dirs = hq[SWQ_REPEND_D];
    out->n_dirty_recs = hq[SWQ_N];
    out->n_dirty_dirs = hq[SWQ_N + 1];
    out->relative_zxid = w.zxid;
    out->frames.n = F;
    out->frames.total = total;
    out->frames.flags = dev_out ? REGK_OUT_DEVICE : 0;
    out->frames.launches = launches;
    out->frames.frame_bytes = (const uint8_t *)src[0];
    out->frames.frame_off = (const uint64_t *)src[1];
    out->frames.kernel_ms = ms;
    return REGK_OK;
}

/* regk_resolve's passes up to the text (shared with regk_walk_resolve): the checks, the insert, decode, classify,
   join, sort, child_len / child_scan and qlen / place passes, and the counters they leave */
struct ResolveRun {
    ResolveParams p;
    uint64_t m = 0, nq = 0, text_total = 0, n_unres = 0, path_total = 0, slots = 0;
    unsigned long long answers = 0, additional = 0;
    bool dev_out = false;
    uint32_t launches = 0;
    float ms = 0;
    const uint8_t *pb = nullptr, *jb = nullptr;
    const uint64_t *po = nullptr, *jo = nullptr;
};

static int resolve_meta(regk_ctx *ctx, const regk_decode_in *in, const regk_resolve_opts *o, const char *who, ResolveRun *run)
{
    if (in->flags & REGK_DECODE_LAST)
        return fail(ctx, REGK_ERR_INVALID_ARG, "%s: REGK_DECODE_LAST names no snapshot; pass the snapshot's streams", who);
    if (o->flags & ~(REGK_OUT_DEVICE | REGK_RESOLVE_ANY_FORM))
        return fail(ctx, REGK_ERR_INVALID_ARG, "%s: unknown flag bits 0x%x", who, o->flags & ~(REGK_OUT_DEVICE | REGK_RESOLVE_ANY_FORM));
    if (o->reserved)
        return fail(ctx, REGK_ERR_INVALID_ARG, "%s: reserved must be 0", who);
    if (o->default_host_ttl < 0 || o->default_srv_ttl < 0)
        return fail(ctx, REGK_ERR_INVALID_ARG, "%s: default TTLs must be >= 0 (host %d, srv %d)", who, o->default_host_ttl,
            o->default_srv_ttl);
    if (ctx->pending)
        return fail(ctx, REGK_ERR_STATE, "%s: batches are still in flight; finish them first", who);
    const uint64_t m = in->n;
    if (m >= 0xFFFFFFFFull)
        return fail(ctx, REGK_ERR_INVALID_ARG, "%s: %llu nodes: must be below 2^32 - 1", who, (unsigned long long)m);
    const bool in_dev = in->flags & REGK_IN_DEVICE, dev_out = o->flags & REGK_OUT_DEVICE;
    const uint8_t *pb = in->path_bytes, *jb = in->json_bytes;
    const uint64_t *po = in->path_off, *jo = in->json_off;
    uint64_t path_total = m ? in->path_total : 0, json_total = m ? in->json_total : 0;
    if (m && (!po || !jo))
        return fail(ctx, REGK_ERR_INVALID_ARG, "%s: a snapshot of %llu nodes needs path and data offsets", who, (unsigned long long)m);
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    regk_ctx::Resolve &rb = ctx->rsv;
    int rc;
    if (m && !in_dev) {
        path_total = po[m];
        json_total = jo[m];
        /* offsets become memory ranges in the kernels: monotone, each node below 4 GiB, ending at the totals */
        for (uint64_t j = 0; j < m; j++)
            if (po[j] > po[j + 1] || jo[j] > jo[j + 1] || po[j + 1] - po[j] > 0xFFFFFFFFull || jo[j + 1] - jo[j] > 0xFFFFFFFFull)
                return fail(ctx, REGK_ERR_INVALID_ARG, "%s: snapshot offsets are not monotone at node %llu", who, (unsigned long long)j);
        if ((path_total && !pb) || (json_total && !jb))
            return fail(ctx, REGK_ERR_INVALID_ARG, "%s: snapshot offsets without bytes", who);
        const void *src[4] = {pb, po, jb, jo};
        const size_t sz[4] = {(size_t)path_total, (size_t)(m + 1) * 8, (size_t)json_total, (size_t)(m + 1) * 8};
        for (int k = 0; k < 4; k++)
            if ((rc = stage_in(ctx, rb.in[k], src[k], sz[k], s)))
                return rc;
        pb = (const uint8_t *)rb.in[0].p;
        po = (const uint64_t *)rb.in[1].p;
        jb = (const uint8_t *)rb.in[2].p;
        jo = (const uint64_t *)rb.in[3].p;
    } else if (m) {
        if ((path_total && !pb) || (json_total && !jb))
            return fail(ctx, REGK_ERR_INVALID_ARG, "%s: snapshot offsets without bytes", who);
        if (((uintptr_t)pb & 3u) || ((uintptr_t)jb & 3u) || ((uintptr_t)po & 7u) || ((uintptr_t)jo & 7u))
            return fail(ctx, REGK_ERR_INVALID_ARG, "%s: misaligned device snapshot (bytes need 4-byte, offsets 8-byte alignment)", who);
    }
    /* an empty stream is never read; its kernels still get a valid pointer */
    if ((rc = ensure_dev(ctx, rb.in[0], 16)) || (rc = ensure_dev(ctx, rb.in[2], 16)))
        return rc;
    if (!pb)
        pb = (const uint8_t *)rb.in[0].p;
    if (!jb)
        jb = (const uint8_t *)rb.in[2].p;
    for (Event &ev : rb.ev)
        if ((rc = ensure_event(ctx, ev)))
            return rc;
    /* sizes: the table at most half full; per-node and per-position arrays; totals of both scans */
    uint64_t slots = 1024;
    while (slots < 2 * m)
        slots <<= 1;
    const uint64_t tiles = (m + RV_TILE - 1) / RV_TILE, nsup = tiles / SUPER + 1;
    const size_t totals_bytes = 6 * (tiles + nsup) * 8;
    const uint32_t end_bit = m ? 32u - (uint32_t)__builtin_clz((uint32_t)m) : 1u;
    size_t sort_bytes = 0;
    CK(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const uint32_t *)nullptr, (uint32_t *)nullptr, (const uint32_t *)nullptr,
        (uint32_t *)nullptr, (int)std::max<uint64_t>(m, 1), 0, (int)end_bit, s));
    if ((rc = ensure_dev(ctx, rb.table, slots * 4)) || (rc = ensure_dev(ctx, rb.slot, m * 4 + 16)) ||
        (rc = ensure_dev(ctx, rb.hash, m * 4 + 16)) || (rc = ensure_dev(ctx, rb.rec, (m + 1) * sizeof(Decoded))) ||
        (rc = ensure_dev(ctx, rb.dom, path_total + 16)) || (rc = ensure_dev(ctx, rb.ports, (json_total / 2 + 1) * 4 + 16)) ||
        (rc = ensure_dev(ctx, rb.cls, m + 16)) || (rc = ensure_dev(ctx, rb.roles, m + 16)) || (rc = ensure_dev(ctx, rb.ttl, m * 4 + 16)) ||
        (rc = ensure_dev(ctx, rb.key, m * 4 + 16)) || (rc = ensure_dev(ctx, rb.val, m * 4 + 16)) ||
        (rc = ensure_dev(ctx, rb.skey, m * 4 + 16)) || (rc = ensure_dev(ctx, rb.sval, m * 4 + 16)) ||
        (rc = ensure_dev(ctx, rb.first, m * 4 + 16)) || (rc = ensure_dev(ctx, rb.end, m * 4 + 16)) ||
        (rc = ensure_dev(ctx, rb.totals, totals_bytes)) || (rc = ensure_dev(ctx, rb.count, RV_NCOUNTERS * 8)) ||
        (rc = ensure_dev(ctx, rb.node_q, m * 8 + 16)) || (rc = ensure_dev(ctx, rb.q_kind, 2 * m + 16)) ||
        (rc = ensure_dev(ctx, rb.q_node, 2 * m * 8 + 16)) || (rc = ensure_dev(ctx, rb.sec_off, (4 * m + 1) * 8)) ||
        (rc = ensure_dev(ctx, rb.unres, m * 8 + 16)) || (rc = ensure_dev(ctx, rb.sort_tmp, sort_bytes + 16)) ||
        (rc = ensure_host(ctx, rb.h_count, RV_NCOUNTERS * 8)))
        return rc;
    for (int k = 0; k < 3; k++)
        if ((rc = ensure_dev(ctx, rb.cum[k], (m + 1) * 8)))
            return rc;
    const bool any = o->flags & REGK_RESOLVE_ANY_FORM;
    if (any && ((rc = ensure_dev(ctx, rb.any_list, m * 4 + 16)) || (rc = ensure_dev(ctx, rb.any_totals, (tiles + nsup) * 8)) ||
                (rc = ensure_dev(ctx, rb.any_count, 16)) || (rc = ensure_host(ctx, rb.h_any, 16))))
        return rc;
    CK(cudaMemsetAsync(rb.table.p, 0, slots * 4, s));
    CK(cudaMemsetAsync(rb.totals.p, 0, totals_bytes, s));
    CK(cudaMemsetAsync(rb.count.p, 0, RV_NCOUNTERS * 8, s));
    CK(cudaMemsetAsync(rb.count.p, 0xFF, 16, s));           /* no bad node, no duplicate node */
    CK(cudaMemsetAsync(rb.first.p, 0, m * 4 + 16, s));      /* a service without children: [0, 0) */
    CK(cudaMemsetAsync(rb.end.p, 0, m * 4 + 16, s));
    CK(cudaMemsetAsync(rb.sec_off.p, 0, 8, s));
    unsigned long long *hc = (unsigned long long *)rb.h_count.p;
    uint32_t launches = 0;
    float ms = 0, part = 0;
    /* 1. offsets check (device snapshots) and every path into the table: regk_reconcile's insert pass */
    ReconcileParams ip{};
    ip.m = m;
    ip.o_path = pb;
    ip.o_path_off = (const unsigned long long *)po;
    ip.o_json = jb;
    ip.o_json_off = (const unsigned long long *)jo;
    ip.o_path_total = path_total;
    ip.o_json_total = json_total;
    ip.validate = in_dev ? 1u : 0u;
    ip.mask_o = (uint32_t)(slots - 1);
    ip.t_obs = (uint32_t *)rb.table.p;
    ip.slot_obs = (uint32_t *)rb.slot.p;
    ip.hash_obs = (uint32_t *)rb.hash.p;
    ip.counters = (unsigned long long *)rb.count.p;
    CK(cudaEventRecord(rb.ev[0], s));
    if (m) {
        regk_reconcile_insert_kernel<<<(unsigned)((m + 255) / 256), 256, 0, s>>>(ip);
        CK(cudaGetLastError());
        launches++;
    }
    CK(cudaEventRecord(rb.ev[1], s));
    if (m && in_dev) {                                      /* the decode pass reads every node's bytes: refuse first */
        CK(cudaMemcpyAsync(hc, rb.count.p, 8, cudaMemcpyDeviceToHost, s));
        if ((rc = sync_or_fail(ctx, s, who)))
            return rc;
        if (hc[RV_C_BAD] != ~0ull)
            return fail(ctx, REGK_ERR_INVALID_ARG, "%s: snapshot offsets are not monotone or reach past the totals at node %llu", who,
                hc[RV_C_BAD]);
    }
    CK(cudaEventRecord(rb.ev[2], s));
    ResolveParams p{};
    p.m = m;
    p.path = pb;
    p.path_off = (const unsigned long long *)po;
    p.json = jb;
    p.json_off = (const unsigned long long *)jo;
    p.path_total = path_total;
    p.dec = (const Decoded *)rb.rec.p;
    p.dom = (const uint8_t *)rb.dom.p;
    p.ports = (const uint32_t *)rb.ports.p;
    p.dflt_host = o->default_host_ttl;
    p.dflt_srv = o->default_srv_ttl;
    p.mask = (uint32_t)(slots - 1);
    p.table = (const uint32_t *)rb.table.p;
    p.slot = (const uint32_t *)rb.slot.p;
    p.cls = (uint8_t *)rb.cls.p;
    p.roles = (uint8_t *)rb.roles.p;
    p.ttl = (int32_t *)rb.ttl.p;
    p.key = (uint32_t *)rb.key.p;
    p.val = (uint32_t *)rb.val.p;
    p.skey = (const uint32_t *)rb.skey.p;
    p.sval = (const uint32_t *)rb.sval.p;
    p.first = (uint32_t *)rb.first.p;
    p.end = (uint32_t *)rb.end.p;
    unsigned long long *tb = (unsigned long long *)rb.totals.p;
    for (int k = 0; k < 3; k++) {
        p.cum[k] = (unsigned long long *)rb.cum[k].p;
        p.ctile[k] = tb + (size_t)k * (tiles + nsup);
        p.csuper[k] = p.ctile[k] + tiles;
        p.ntile[k] = tb + (size_t)(3 + k) * (tiles + nsup);
        p.nsuper[k] = p.ntile[k] + tiles;
    }
    p.node_q = (unsigned long long *)rb.node_q.p;
    p.q_kind = (uint8_t *)rb.q_kind.p;
    p.q_node = (unsigned long long *)rb.q_node.p;
    p.sec_off = (unsigned long long *)rb.sec_off.p;
    p.unresolved = (unsigned long long *)rb.unres.p;
    p.counters = (unsigned long long *)rb.count.p;
    if (m) {
        /* 2. decode (host_nodes = 0): regk_decode's kernel and staging budgets */
        DecodeParams dp{};
        dp.n = m;
        dp.path_bytes = pb;
        dp.path_off = (const unsigned long long *)po;
        dp.json_bytes = jb;
        dp.json_off = (const unsigned long long *)jo;
        dp.host_nodes = 0;
        dp.out = (Decoded *)rb.rec.p;
        dp.dom_bytes = (uint8_t *)rb.dom.p;
        dp.ports = (uint32_t *)rb.ports.p;
        dp.path_cap = (uint32_t)align16(std::min<uint64_t>(path_total * DEC_TILE / m * 9 / 8 + 1024, 49152));
        dp.json_cap = (uint32_t)align16(std::min<uint64_t>(json_total * DEC_TILE / m * 9 / 8 + 1024, 65536));
        const uint64_t slack = in_dev ? 0 : 16;             /* a caller's own device buffers end where they end */
        dp.path_limit = path_total + slack;
        dp.json_limit = json_total + slack;
        const size_t dsmem = std::max<size_t>((size_t)dp.path_cap + 32, DEC_TILE * sizeof(Decoded)) + ((dp.path_cap / 8 + 47) & ~15u) +
            std::max<size_t>(dp.json_cap, dp.path_cap) + 32 + 16;
        if ((rc = set_smem_limit(ctx, (const void *)regk_decode_kernel, dsmem)))
            return rc;
        regk_decode_kernel<<<(unsigned)((m + DEC_TILE - 1) / DEC_TILE), DEC_TILE, dsmem, s>>>(dp);
        const unsigned g256 = (unsigned)((m + 255) / 256);
        if (any) {
            /* 2b. REGK_RESOLVE_ANY_FORM: the candidates in node order, then the general reader over them */
            AnyParams ap{};
            ap.m = m;
            ap.json = jb;
            ap.json_off = (const unsigned long long *)jo;
            ap.json_limit = dp.json_limit;
            ap.dec = (Decoded *)rb.rec.p;
            ap.ports = (uint32_t *)rb.ports.p;
            ap.list = (uint32_t *)rb.any_list.p;
            for (int k = 0; k < 3; k++) {
                ap.tile_total[k] = (unsigned long long *)rb.any_totals.p;
                ap.super_total[k] = ap.tile_total[k] + tiles;
            }
            ap.count = (unsigned long long *)rb.any_count.p;
            CK(cudaMemsetAsync(rb.any_totals.p, 0, (tiles + nsup) * 8, s));
            regk_resolve_any_count_kernel<<<(unsigned)tiles, RV_TILE, 0, s>>>(ap);
            regk_resolve_any_compact_kernel<<<(unsigned)tiles, RV_TILE, 0, s>>>(ap);
            CK(cudaGetLastError());
            launches += 2;
            unsigned long long *hn = (unsigned long long *)rb.h_any.p;
            CK(cudaMemcpyAsync(hn, rb.any_count.p, 8, cudaMemcpyDeviceToHost, s));
            if ((rc = sync_or_fail(ctx, s, who)))
                return rc;
            if (*hn) {
                regk_resolve_any_read_kernel<<<(unsigned)((*hn + 255) / 256), 256, 0, s>>>(ap, (uint32_t)*hn);
                CK(cudaGetLastError());
                launches++;
            }
        }
        /* 3. classify, 4. join, 5. group, 6. size and place */
        if (any)
            regk_resolve_classify_any_kernel<<<g256, 256, 0, s>>>(p);
        else
            regk_resolve_classify_kernel<<<g256, 256, 0, s>>>(p);
        regk_resolve_join_kernel<<<g256, 256, 0, s>>>(p);
        CK(cudaGetLastError());
        size_t tmp = rb.sort_tmp.cap;
        CK(cub::DeviceRadixSort::SortPairs(rb.sort_tmp.p, tmp, (const uint32_t *)p.key, (uint32_t *)rb.skey.p, (const uint32_t *)p.val,
            (uint32_t *)rb.sval.p, (int)m, 0, (int)end_bit, s));
        regk_resolve_child_len_kernel<<<(unsigned)tiles, RV_TILE, 0, s>>>(p);
        regk_resolve_child_scan_kernel<<<(unsigned)tiles, RV_TILE, 0, s>>>(p);
        regk_resolve_qlen_kernel<<<(unsigned)tiles, RV_TILE, 0, s>>>(p);
        regk_resolve_place_kernel<<<(unsigned)tiles, RV_TILE, 0, s>>>(p);
        CK(cudaGetLastError());
        launches += 8;                                      /* the radix sort counted as one */
    }
    CK(cudaEventRecord(rb.ev[3], s));
    CK(cudaMemcpyAsync(hc, rb.count.p, RV_NCOUNTERS * 8, cudaMemcpyDeviceToHost, s));
    if ((rc = sync_or_fail(ctx, s, who)))
        return rc;
    if (m && hc[RV_C_DUP] != ~0ull)
        return fail(ctx, REGK_ERR_INVALID_ARG, "%s: snapshot node %llu has the path of an earlier node; a registry cannot "
                                               "hold two nodes with one path", who, hc[RV_C_DUP]);
    cudaEventElapsedTime(&ms, rb.ev[0], rb.ev[1]);
    cudaEventElapsedTime(&part, rb.ev[2], rb.ev[3]);
    ms += part;
    run->p = p;
    run->m = m;
    run->nq = m ? hc[RV_C_QUERIES] : 0;
    run->text_total = m ? hc[RV_C_TEXT] : 0;
    run->n_unres = m ? hc[RV_C_UNRESOLVED] : 0;
    run->answers = m ? hc[RV_C_ANSWERS] : 0;
    run->additional = m ? hc[RV_C_ADDITIONAL] : 0;
    run->path_total = path_total;
    run->slots = slots;
    run->dev_out = dev_out;
    run->launches = launches;
    run->ms = ms;
    run->pb = pb;
    run->po = po;
    run->jb = jb;
    run->jo = jo;
    return REGK_OK;
}

/* The answers of a resolve whose text is `text` (device): copied out unless REGK_OUT_DEVICE, kernel_ms adding the
   events [a, b), and the state regk_dns_answer answers from. */
static int resolve_publish(regk_ctx *ctx, const ResolveRun &r, const void *text, cudaEvent_t a, cudaEvent_t b, regk_answers *out,
    const char *who)
{
    regk_ctx::Resolve &rb = ctx->rsv;
    cudaStream_t s = ctx->stream;
    int rc;
    const uint64_t m = r.m, nq = r.nq;
    const void *dsrc[6] = {rb.q_kind.p, rb.q_node.p, rb.sec_off.p, text, rb.cls.p, rb.unres.p};
    if (!r.dev_out) {
        HostBuf *hb[6] = {&rb.h_q_kind, &rb.h_q_node, &rb.h_sec_off, &rb.h_text, &rb.h_cls, &rb.h_unres};
        const size_t sz[6] = {(size_t)nq, (size_t)nq * 8, (size_t)(2 * nq + 1) * 8, (size_t)r.text_total, (size_t)m,
                              (size_t)r.n_unres * 8};
        for (int k = 0; k < 6; k++) {
            if ((rc = to_host(ctx, *hb[k], dsrc[k], sz[k], s)))
                return rc;
            dsrc[k] = hb[k]->p;
        }
    }
    if ((rc = sync_or_fail(ctx, s, who)))
        return rc;
    float part = 0;
    cudaEventElapsedTime(&part, a, b);
    out->m = m;
    out->n_queries = nq;
    out->n_answers = r.answers;
    out->n_additional = r.additional;
    out->n_unresolved = r.n_unres;
    out->text_total = r.text_total;
    out->flags = r.dev_out ? REGK_OUT_DEVICE : 0;
    out->launches = r.launches;
    out->q_kind = (const uint8_t *)dsrc[0];
    out->q_node = (const uint64_t *)dsrc[1];
    out->sec_off = (const uint64_t *)dsrc[2];
    out->text = (const uint8_t *)dsrc[3];
    out->node_cls = (const uint8_t *)dsrc[4];
    out->unresolved = (const uint64_t *)dsrc[5];
    out->kernel_ms = r.ms + part;
    rb.valid = true;
    rb.walk = false;
    rb.gen++;
    rb.m = m;
    rb.path_total = r.path_total;
    rb.slots = r.slots;
    rb.pb = r.pb;
    rb.po = r.po;
    rb.jb = r.jb;
    rb.jo = r.jo;
    return REGK_OK;
}

int regk_resolve(regk_ctx *ctx, const regk_decode_in *in, const regk_resolve_opts *o, regk_answers *out)
{
    const char *who = "regk_resolve";
    if (!ctx || !in || !o || !out)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_resolve: NULL argument");
    memset(out, 0, sizeof *out);
    ctx->rsv.valid = false;
    ResolveRun r;
    int rc;
    if ((rc = resolve_meta(ctx, in, o, who, &r)))
        return rc;
    regk_ctx::Resolve &rb = ctx->rsv;
    cudaStream_t s = ctx->stream;
    /* 7. emit */
    if ((rc = ensure_dev(ctx, rb.text, r.text_total + 16)))
        return rc;
    r.p.text = (uint8_t *)rb.text.p;
    CK(cudaEventRecord(rb.ev[3], s));
    if (r.m && r.text_total) {
        regk_resolve_emit_kernel<<<(unsigned)((2 * r.m + 255) / 256), 256, 0, s>>>(r.p);
        CK(cudaGetLastError());
        r.launches++;
    }
    CK(cudaEventRecord(rb.ev[4], s));
    return resolve_publish(ctx, r, rb.text.p, rb.ev[3], rb.ev[4], out, who);
}

int regk_dns_answer(regk_ctx *ctx, const regk_dns_in *in, const regk_dns_opts *o, regk_dns_out *out)
{
    const char *who = "regk_dns_answer";
    if (!ctx || !in || !o || !out)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_dns_answer: NULL argument");
    memset(out, 0, sizeof *out);
    if (in->flags & ~REGK_IN_DEVICE)
        return fail(ctx, REGK_ERR_INVALID_ARG, "%s: unknown input flag bits 0x%x", who, in->flags & ~REGK_IN_DEVICE);
    if (in->reserved)
        return fail(ctx, REGK_ERR_INVALID_ARG, "%s: reserved must be 0", who);
    if (o->flags & ~(REGK_OUT_DEVICE | REGK_DNS_TCP | REGK_DNS_PTR))
        return fail(ctx, REGK_ERR_INVALID_ARG, "%s: unknown flag bits 0x%x", who,
            o->flags & ~(REGK_OUT_DEVICE | REGK_DNS_TCP | REGK_DNS_PTR));
    if (o->udp_payload < 512u || o->udp_payload > 65535u)
        return fail(ctx, REGK_ERR_INVALID_ARG, "%s: udp_payload %u outside 512..65535", who, o->udp_payload);
    const regk_ctx::Resolve &rb = ctx->rsv;
    if (!rb.valid)
        return fail(ctx, REGK_ERR_STATE, "%s: no successful regk_resolve on this context to answer from", who);
    if (rb.walk && rb.walk_sgen != ctx->wk.sgen)
        return fail(ctx, REGK_ERR_STATE, "%s: the walk's snapshot changed since regk_walk_resolve; resolve it again "
                                         "(regk_walk_resolve) before answering", who);
    if (ctx->pending)
        return fail(ctx, REGK_ERR_STATE, "%s: batches are still in flight; finish them first", who);
    const uint64_t k = in->k, m = rb.m;
    const bool in_dev = in->flags & REGK_IN_DEVICE, dev_out = o->flags & REGK_OUT_DEVICE, ptr = o->flags & REGK_DNS_PTR;
    if (k && !in->off)
        return fail(ctx, REGK_ERR_INVALID_ARG, "%s: %llu messages need offsets", who, (unsigned long long)k);
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    regk_ctx::Dns &db = ctx->dns;
    int rc;
    uint64_t total = k ? in->total : 0;
    const uint8_t *mb = in->msgs;
    const uint64_t *mo = in->off;
    if (k && !in_dev) {
        total = mo[k];
        for (uint64_t i = 0; i < k; i++)
            if (mo[i] > mo[i + 1] || mo[i + 1] > total || mo[i + 1] - mo[i] > 65535u)
                return fail(ctx, REGK_ERR_INVALID_ARG, "%s: message %llu: offsets not monotone, past total or longer than 65535 "
                                                       "bytes", who, (unsigned long long)i);
        if (total && !mb)
            return fail(ctx, REGK_ERR_INVALID_ARG, "%s: offsets without message bytes", who);
        if ((rc = stage_in(ctx, db.in[0], mb, total, s)) || (rc = stage_in(ctx, db.in[1], mo, (k + 1) * 8, s)))
            return rc;
        mb = (const uint8_t *)db.in[0].p;
        mo = (const uint64_t *)db.in[1].p;
    } else if (k) {
        if (total && !mb)
            return fail(ctx, REGK_ERR_INVALID_ARG, "%s: offsets without message bytes", who);
        if ((uintptr_t)mo & 7u)
            return fail(ctx, REGK_ERR_INVALID_ARG, "%s: misaligned device offsets (8-byte alignment)", who);
    }
    if ((rc = ensure_dev(ctx, db.in[0], 16)))
        return rc;
    if (!mb)
        mb = (const uint8_t *)db.in[0].p;
    for (Event &ev : db.ev)
        if ((rc = ensure_event(ctx, ev)))
            return rc;
    const uint64_t ptiles = (m + RV_TILE - 1) / RV_TILE, pnsup = ptiles / SUPER + 1;
    const uint64_t tiles = (k + RV_TILE - 1) / RV_TILE, nsup = tiles / SUPER + 1;
    if ((rc = ensure_dev(ctx, db.ip4, m * 4 + 16)) || (rc = ensure_dev(ctx, db.ptotals, 3 * (ptiles + pnsup) * 8)) ||
        (rc = ensure_dev(ctx, db.scratch, total + 16)) || (rc = ensure_dev(ctx, db.status, k + 16)) ||
        (rc = ensure_dev(ctx, db.tc, k + 16)) || (rc = ensure_dev(ctx, db.node, k * 8 + 16)) ||
        (rc = ensure_dev(ctx, db.meta, k * 4 + 16)) || (rc = ensure_dev(ctx, db.nans, k * 4 + 16)) ||
        (rc = ensure_dev(ctx, db.nadd, k * 4 + 16)) || (rc = ensure_dev(ctx, db.ans_bytes, k * 4 + 16)) ||
        (rc = ensure_dev(ctx, db.qtotals, 2 * (tiles + nsup) * 8)) || (rc = ensure_dev(ctx, db.resp_off, (k + 1) * 8)) ||
        (rc = ensure_dev(ctx, db.rr_base, (k + 1) * 8)) || (rc = ensure_dev(ctx, db.count, DNS_NCOUNTERS * 8)) ||
        (rc = ensure_host(ctx, db.h_count, DNS_NCOUNTERS * 8)))
        return rc;
    for (int j = 0; j < 3; j++)
        if ((rc = ensure_dev(ctx, db.cum[j], (m + 1) * 8)))
            return rc;
    /* the reverse index, sized for every node a host node */
    const bool build_ptr = ptr && db.ptr_gen != rb.gen;
    if (build_ptr) {
        db.ptr_gen = 0;
        size_t sort_bytes = 0;
        CK(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const uint32_t *)nullptr, (uint32_t *)nullptr,
            (const uint32_t *)nullptr, (uint32_t *)nullptr, (int)std::max<uint64_t>(m, 1), 0, 32, s));
        if ((rc = ensure_dev(ctx, db.pkey_in, m * 4 + 16)) || (rc = ensure_dev(ctx, db.pval_in, m * 4 + 16)) ||
            (rc = ensure_dev(ctx, db.pkey, m * 4 + 16)) || (rc = ensure_dev(ctx, db.pval, m * 4 + 16)) ||
            (rc = ensure_dev(ctx, db.pbytes, (m + 1) * 8)) || (rc = ensure_dev(ctx, db.ptr_tmp, sort_bytes + 16)) ||
            (rc = ensure_dev(ctx, db.ptr_totals, 2 * (ptiles + pnsup) * 8)) || (rc = ensure_dev(ctx, db.ptr_count, 16)))
            return rc;
    }
    DnsParams p{};
    p.m = m;
    p.path = rb.pb;
    p.path_off = (const unsigned long long *)rb.po;
    p.path_total = rb.path_total;
    p.json = rb.jb;
    p.json_off = (const unsigned long long *)rb.jo;
    p.dec = (const Decoded *)rb.rec.p;
    p.dom = (const uint8_t *)rb.dom.p;
    p.ports = (const uint32_t *)rb.ports.p;
    p.mask = (uint32_t)(rb.slots - 1);
    p.table = (const uint32_t *)rb.table.p;
    p.cls = (const uint8_t *)rb.cls.p;
    p.roles = (const uint8_t *)rb.roles.p;
    p.ttl = (const int32_t *)rb.ttl.p;
    p.skey = (const uint32_t *)rb.skey.p;
    p.sval = (const uint32_t *)rb.sval.p;
    p.first = (const uint32_t *)rb.first.p;
    p.end = (const uint32_t *)rb.end.p;
    p.ip4 = (uint32_t *)db.ip4.p;
    unsigned long long *pt = (unsigned long long *)db.ptotals.p, *qt = (unsigned long long *)db.qtotals.p;
    for (int j = 0; j < 3; j++) {
        p.cum[j] = (unsigned long long *)db.cum[j].p;
        p.ctile[j] = pt + (size_t)j * (ptiles + pnsup);
        p.csuper[j] = p.ctile[j] + ptiles;
        p.qtile[j] = qt + (size_t)(j < 2 ? j : 1) * (tiles + nsup);
        p.qsuper[j] = p.qtile[j] + tiles;
    }
    p.k = k;
    p.msgs = mb;
    p.off = (const unsigned long long *)mo;
    p.total = total;
    p.scratch = (uint8_t *)db.scratch.p;
    p.udp_payload = o->udp_payload;
    p.tcp = (o->flags & REGK_DNS_TCP) ? 1u : 0u;
    p.status = (uint8_t *)db.status.p;
    p.tc = (uint8_t *)db.tc.p;
    p.node = (unsigned long long *)db.node.p;
    p.meta = (uint32_t *)db.meta.p;
    p.nans = (uint32_t *)db.nans.p;
    p.nadd = (uint32_t *)db.nadd.p;
    p.ans_bytes = (uint32_t *)db.ans_bytes.p;
    p.resp_off = (unsigned long long *)db.resp_off.p;
    p.rr_base = (unsigned long long *)db.rr_base.p;
    p.counters = (unsigned long long *)db.count.p;
    DnsPtrParams x{};
    x.n = db.ptr_n;
    x.key = x.skey = (uint32_t *)db.pkey.p;
    x.val = x.sval = (uint32_t *)db.pval.p;
    x.bytes = x.sbytes = (unsigned long long *)db.pbytes.p;
    x.key_in = (uint32_t *)db.pkey_in.p;
    x.val_in = (uint32_t *)db.pval_in.p;
    x.htile[0] = (unsigned long long *)db.ptr_totals.p;
    x.hsuper[0] = x.htile[0] + ptiles;
    x.btile[0] = x.hsuper[0] + pnsup;
    x.bsuper[0] = x.btile[0] + ptiles;
    x.count = (unsigned long long *)db.ptr_count.p;
    unsigned long long *hc = (unsigned long long *)db.h_count.p;
    uint32_t launches = 0;
    float ms = 0, part = 0;
    CK(cudaMemsetAsync(db.count.p, 0, DNS_NCOUNTERS * 8, s));
    CK(cudaMemsetAsync(db.count.p, 0xFF, 8, s));            /* no bad message */
    CK(cudaMemsetAsync(db.qtotals.p, 0, 2 * (tiles + nsup) * 8, s));
    CK(cudaMemsetAsync(db.resp_off.p, 0, 8, s));
    CK(cudaMemsetAsync(db.rr_base.p, 0, 8, s));
    CK(cudaEventRecord(db.ev[0], s));
    /* 1. once per resolve: addresses and the per-child wire sizes */
    if (db.prep_gen != rb.gen) {
        CK(cudaMemsetAsync(db.ptotals.p, 0, 3 * (ptiles + pnsup) * 8, s));
        CK(cudaMemsetAsync(db.cum[0].p, 0, 8, s));
        CK(cudaMemsetAsync(db.cum[1].p, 0, 8, s));
        CK(cudaMemsetAsync(db.cum[2].p, 0, 8, s));
        if (m) {
            regk_dns_prep_kernel<<<(unsigned)ptiles, RV_TILE, 0, s>>>(p);
            regk_dns_prep_scan_kernel<<<(unsigned)ptiles, RV_TILE, 0, s>>>(p);
            CK(cudaGetLastError());
            launches += 2;
        }
    }
    /* 1b. once per resolve with REGK_DNS_PTR: the reverse index (its count read back to size the sort) */
    if (build_ptr) {
        CK(cudaMemsetAsync(db.ptr_totals.p, 0, 2 * (ptiles + pnsup) * 8, s));
        CK(cudaMemsetAsync(db.ptr_count.p, 0, 8, s));
        CK(cudaMemsetAsync(db.pbytes.p, 0, 8, s));
        if (m) {
            regk_dns_ptr_count_kernel<<<(unsigned)ptiles, RV_TILE, 0, s>>>(p, x);
            regk_dns_ptr_compact_kernel<<<(unsigned)ptiles, RV_TILE, 0, s>>>(p, x);
            CK(cudaGetLastError());
            launches += 2;
        }
        CK(cudaEventRecord(db.ev[1], s));
        CK(cudaMemcpyAsync(hc, db.ptr_count.p, 8, cudaMemcpyDeviceToHost, s));
        if ((rc = sync_or_fail(ctx, s, who)))
            return rc;
        cudaEventElapsedTime(&part, db.ev[0], db.ev[1]);
        ms += part;
        CK(cudaEventRecord(db.ev[0], s));
        x.n = hc[0];
        if (x.n) {
            const uint64_t btiles = (x.n + RV_TILE - 1) / RV_TILE;
            size_t tmp = db.ptr_tmp.cap;
            CK(cub::DeviceRadixSort::SortPairs(db.ptr_tmp.p, tmp, (const uint32_t *)x.key_in, x.skey, (const uint32_t *)x.val_in,
                x.sval, (int)x.n, 0, 32, s));
            regk_dns_ptr_len_kernel<<<(unsigned)btiles, RV_TILE, 0, s>>>(p, x);
            regk_dns_ptr_scan_kernel<<<(unsigned)btiles, RV_TILE, 0, s>>>(p, x);
            CK(cudaGetLastError());
            launches += 3;                                  /* the radix sort counted as one */
        }
    }
    /* 2. device offsets, before any message byte is read */
    if (k && in_dev) {
        regk_dns_check_kernel<<<(unsigned)((k + 255) / 256), 256, 0, s>>>(p);
        CK(cudaGetLastError());
        launches++;
        CK(cudaEventRecord(db.ev[1], s));
        CK(cudaMemcpyAsync(hc, db.count.p, 8, cudaMemcpyDeviceToHost, s));
        if ((rc = sync_or_fail(ctx, s, who)))
            return rc;
        if (hc[DNS_C_BAD] != ~0ull)
            return fail(ctx, REGK_ERR_INVALID_ARG, "%s: message %llu: offsets not monotone, past total or longer than 65535 bytes",
                who, hc[DNS_C_BAD]);
        cudaEventElapsedTime(&part, db.ev[0], db.ev[1]);
        ms += part;
        CK(cudaEventRecord(db.ev[0], s));
    }
    db.prep_gen = rb.gen;
    /* 3. parse, look up and cut; 4. place */
    if (k) {
        if (ptr)
            regk_dns_parse_ptr_kernel<<<(unsigned)tiles, RV_TILE, 0, s>>>(p, x);
        else
            regk_dns_parse_kernel<<<(unsigned)tiles, RV_TILE, 0, s>>>(p);
        regk_dns_place_kernel<<<(unsigned)tiles, RV_TILE, 0, s>>>(p);
        CK(cudaGetLastError());
        launches += 2;
    }
    CK(cudaEventRecord(db.ev[1], s));
    CK(cudaMemcpyAsync(hc, db.count.p, DNS_NCOUNTERS * 8, cudaMemcpyDeviceToHost, s));
    if ((rc = sync_or_fail(ctx, s, who)))
        return rc;
    cudaEventElapsedTime(&part, db.ev[0], db.ev[1]);
    ms += part;
    const uint64_t resp_total = k ? hc[DNS_C_RESP] : 0, n_rr = k ? hc[DNS_C_RR] : 0;
    /* 5. emit */
    if ((rc = ensure_dev(ctx, db.resp, resp_total + 16)))
        return rc;
    p.resp = (uint8_t *)db.resp.p;
    CK(cudaEventRecord(db.ev[2], s));
    if (resp_total) {
        regk_dns_emit_head_kernel<<<(unsigned)((k + 255) / 256), 256, 0, s>>>(p);
        launches++;
        if (n_rr) {
            if (ptr)
                regk_dns_emit_rr_ptr_kernel<<<(unsigned)((n_rr + 255) / 256), 256, 0, s>>>(p, n_rr, x);
            else
                regk_dns_emit_rr_kernel<<<(unsigned)((n_rr + 255) / 256), 256, 0, s>>>(p, n_rr);
            launches++;
        }
        CK(cudaGetLastError());
    }
    CK(cudaEventRecord(db.ev[3], s));
    const void *dsrc[5] = {db.resp_off.p, db.resp.p, db.status.p, db.tc.p, db.node.p};
    if (!dev_out) {
        HostBuf *hb[5] = {&db.h_resp_off, &db.h_resp, &db.h_status, &db.h_tc, &db.h_node};
        const size_t sz[5] = {(size_t)(k + 1) * 8, (size_t)resp_total, (size_t)k, (size_t)k, (size_t)k * 8};
        for (int j = 0; j < 5; j++) {
            if ((rc = to_host(ctx, *hb[j], dsrc[j], sz[j], s)))
                return rc;
            dsrc[j] = hb[j]->p;
        }
    }
    if ((rc = sync_or_fail(ctx, s, who)))
        return rc;
    cudaEventElapsedTime(&part, db.ev[2], db.ev[3]);
    ms += part;
    out->k = k;
    out->resp_total = resp_total;
    for (int j = 0; j < 8; j++)
        out->n_status[j] = k ? hc[DNS_C_STATUS + j] : 0;
    out->n_truncated = k ? hc[DNS_C_TC] : 0;
    out->flags = dev_out ? REGK_OUT_DEVICE : 0;
    out->launches = launches;
    out->resp_off = (const uint64_t *)dsrc[0];
    out->resp = (const uint8_t *)dsrc[1];
    out->status = (const uint8_t *)dsrc[2];
    out->tc = (const uint8_t *)dsrc[3];
    out->node = (const uint64_t *)dsrc[4];
    out->kernel_ms = ms;
    if (build_ptr) {
        db.ptr_gen = rb.gen;
        db.ptr_n = x.n;
    }
    return REGK_OK;
}

/* `b` grown to hold `need` bytes with its first `used` kept: at least doubled, so that the levels of a walk are copied
   O(log levels) times in all */
static int walk_grow(regk_ctx *ctx, DevBuf &b, size_t used, size_t need)
{
    if (need <= b.cap)
        return REGK_OK;
    DevBuf nb;
    size_t want = (std::max(need, 2 * b.cap) + 255) & ~(size_t)255;
    cudaError_t e = cudaMalloc(&nb.p, want);
    if (e != cudaSuccess) {
        cudaGetLastError();
        want = (need + 255) & ~(size_t)255;
        e = cudaMalloc(&nb.p, want);
    }
    if (e != cudaSuccess)
        return fail(ctx, REGK_ERR_NOMEM, "cudaMalloc(%zu) failed: %s", want, cudaGetErrorString(e));
    nb.cap = want;
    if (used)
        CK(cudaMemcpyAsync(nb.p, b.p, used, cudaMemcpyDeviceToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    std::swap(b, nb);                           /* nb now holds the old buffer and frees it */
    return REGK_OK;
}

/* The walk's path table over its current snapshot (regk_walk_insert_kernel: node + 1 under the hash of its path).  A
   table stays valid while the snapshot only grows (rgen counts the rebuilds, which renumber nodes): the nodes appended
   since it was built are inserted while the table still has twice as many slots as nodes, else it is built anew.
   *built = the nodes inserted this call (0: it was current). */
static int walk_table(regk_ctx *ctx, uint64_t *built, uint32_t *launches, const char *who)
{
    regk_ctx::Walk &wk = ctx->wk;
    cudaStream_t s = ctx->stream;
    const uint64_t m = wk.m;
    int rc;
    *built = 0;
    const bool valid = wk.tab_valid && wk.tab_rgen == wk.rgen;
    if (valid && wk.tab_m == m)
        return REGK_OK;
    uint64_t j0 = 0;
    if (valid && 2 * m <= (uint64_t)wk.tab_mask + 1) {
        j0 = wk.tab_m;
    } else {
        uint64_t sr = 1024;
        while (sr < 2 * m)
            sr <<= 1;
        if (sr > (1ull << 32))
            return fail(ctx, REGK_ERR_INVALID_ARG, "%s: a snapshot of %llu nodes is too large for one table", who,
                (unsigned long long)m);
        if ((rc = ensure_dev(ctx, wk.table, sr * 4)))
            return rc;
        CK(cudaMemsetAsync(wk.table.p, 0, sr * 4, s));
        wk.tab_mask = (uint32_t)(sr - 1);
    }
    if (m > j0) {
        regk_walk_insert_kernel<<<(unsigned)((m - j0 + 255) / 256), 256, 0, s>>>((uint32_t *)wk.table.p, wk.tab_mask,
            (const uint8_t *)wk.snap_bytes[0].p, (const unsigned long long *)wk.snap_off[0].p, j0, m);
        CK(cudaGetLastError());
        (*launches)++;
    }
    wk.tab_m = m;
    wk.tab_rgen = wk.rgen;
    wk.tab_valid = true;
    *built = m - j0;
    return REGK_OK;
}

/* Every buffer walk_filter needs for n listed paths of `total` bytes, so that it cannot fail on an allocation once a
   refresh level's replies have been applied (pack_strings then finds its buffers large enough). */
static int walk_filter_reserve(regk_ctx *ctx, uint64_t n, uint64_t total)
{
    regk_ctx::Walk &wk = ctx->wk;
    const uint64_t tiles = (n + RP_TILE - 1) / RP_TILE, gt = (n + MK_TILE - 1) / MK_TILE;
    const size_t tb = align16(tiles * 4) + (tiles / SUPER + 1) * 8;
    int rc;
    if ((rc = ensure_dev(ctx, wk.xtotals, tb)) || (rc = ensure_dev(ctx, wk.xkeep, n + 16)) ||
        (rc = ensure_dev(ctx, wk.xrec, n * 8 + 16)) || (rc = ensure_dev(ctx, wk.xlen, n * 4 + 16)) ||
        (rc = ensure_dev(ctx, wk.xcount, 16)) || (rc = ensure_dev(ctx, wk.gtotals, gt * 8 + (gt / SUPER + 1) * 8 + 16)) ||
        (rc = ensure_dev(ctx, wk.xoff, (n + 1) * 8)) || (rc = ensure_dev(ctx, wk.xbytes, total + 16)))
        return rc;
    return REGK_OK;
}

/* Every buffer walk_rebuild needs for the current snapshot, whose data may take up to `extra` more bytes from a reply
   stream. */
static int walk_rebuild_reserve(regk_ctx *ctx, uint64_t extra)
{
    regk_ctx::Walk &wk = ctx->wk;
    const uint64_t m = wk.m, tiles = (m + RP_TILE - 1) / RP_TILE, gt = (m + MK_TILE - 1) / MK_TILE;
    const size_t tb = align16(tiles * 4) + (tiles / SUPER + 1) * 8;
    const size_t m8 = m * 8 + 16, m4 = m * 4 + 16;
    int rc;
    if ((rc = ensure_dev(ctx, wk.ktotals, tb)) || (rc = ensure_dev(ctx, wk.kcount, 16)) || (rc = ensure_dev(ctx, wk.psrc, m8)) ||
        (rc = ensure_dev(ctx, wk.dsrc, m8)) || (rc = ensure_dev(ctx, wk.kplen, m4)) || (rc = ensure_dev(ctx, wk.kdlen, m4)) ||
        (rc = ensure_dev(ctx, wk.dsel, m + 16)) || (rc = ensure_dev(ctx, wk.wmark2, m4)) || (rc = ensure_dev(ctx, wk.ver2, m4)) ||
        (rc = ensure_dev(ctx, wk.own2, m8)) || (rc = ensure_dev(ctx, wk.rpos, m8)) || (rc = ensure_dev(ctx, wk.rlen, m4)) ||
        (rc = ensure_dev(ctx, wk.gtotals, gt * 8 + (gt / SUPER + 1) * 8 + 16)) || (rc = ensure_dev(ctx, wk.armed2, m + 16)) ||
        (rc = ensure_dev(ctx, wk.ident2, m4)))
        return rc;
    const uint64_t bytes[2] = {wk.path_total, wk.data_total + extra};
    for (int g = 0; g < 2; g++)
        if ((rc = ensure_dev(ctx, wk.snap2_off[g], (m + 1) * 8 + 16)) || (rc = ensure_dev(ctx, wk.snap2_bytes[g], bytes[g] + 16)))
            return rc;
    return REGK_OK;
}

/* The n listed paths of frontier set nx without those the snapshot holds (skip_removed: holds unmarked), repacked in
   listing order as that frontier; *kept / *total = the entries and bytes left. */
static int walk_filter(regk_ctx *ctx, int nx, uint64_t n, bool skip_removed, uint64_t *kept, uint64_t *total,
    uint32_t *launches, const char *who)
{
    regk_ctx::Walk &wk = ctx->wk;
    cudaStream_t s = ctx->stream;
    uint64_t built;
    int rc;
    if ((rc = walk_table(ctx, &built, launches, who)) || (rc = walk_filter_reserve(ctx, n, *total)))
        return rc;
    const uint64_t tiles = (n + RP_TILE - 1) / RP_TILE;
    const size_t tb = align16(tiles * 4) + (tiles / SUPER + 1) * 8;
    WalkFilterParams fp{};
    fp.n = n;
    fp.lbytes = (const uint8_t *)wk.fbytes[nx].p;
    fp.loff = (const unsigned long long *)wk.foff[nx].p;
    fp.ltotal = *total;
    fp.spath = (const uint8_t *)wk.snap_bytes[0].p;
    fp.soff = (const unsigned long long *)wk.snap_off[0].p;
    fp.table = (const uint32_t *)wk.table.p;
    fp.mask = wk.tab_mask;
    fp.mark = (const uint32_t *)wk.wmark.p;
    fp.skip_removed = skip_removed ? 1u : 0u;
    fp.tile_total = (uint32_t *)wk.xtotals.p;
    fp.super_total = (unsigned long long *)((uint8_t *)wk.xtotals.p + align16(tiles * 4));
    fp.keep = (uint8_t *)wk.xkeep.p;
    fp.rec = (unsigned long long *)wk.xrec.p;
    fp.len = (uint32_t *)wk.xlen.p;
    fp.count = (unsigned long long *)wk.xcount.p;
    CK(cudaMemsetAsync(wk.xtotals.p, 0, tb, s));
    regk_walk_filter_count_kernel<<<(unsigned)tiles, RP_TILE, 0, s>>>(fp);
    regk_walk_filter_kernel<<<(unsigned)tiles, RP_TILE, 0, s>>>(fp);
    CK(cudaGetLastError());
    *launches += 2;
    unsigned long long k = 0;
    CK(cudaMemcpyAsync(&k, fp.count, 8, cudaMemcpyDeviceToHost, s));
    if ((rc = sync_or_fail(ctx, s, who)))
        return rc;
    if ((rc = pack_strings(ctx, k, fp.lbytes, fp.loff, fp.rec, fp.len, wk.gtotals, wk.xbytes, wk.xoff, total, launches)))
        return rc;
    if (k)
        CK(cudaMemcpyAsync(wk.flen[nx].p, fp.len, k * 4, cudaMemcpyDeviceToDevice, s));
    std::swap(wk.fbytes[nx], wk.xbytes);
    std::swap(wk.foff[nx], wk.xoff);
    *kept = k;
    return REGK_OK;
}

/* n items (item k: len[k] bytes at src_off[k] of src1 where sel[k], else of src0) packed into bytes / off by
   regk_mkdirp_len_kernel's totals and the rebuild gather; *total = their bytes. */
static int walk_pack(regk_ctx *ctx, uint64_t n, const uint8_t *src0, const uint8_t *src1, const unsigned long long *src_off,
    const uint8_t *sel, const uint32_t *len, DevBuf &bytes, DevBuf &off, uint64_t *total, uint32_t *launches)
{
    regk_ctx::Walk &wk = ctx->wk;
    cudaStream_t s = ctx->stream;
    const uint64_t gt = (n + MK_TILE - 1) / MK_TILE;
    int rc;
    *total = 0;
    if ((rc = ensure_dev(ctx, wk.gtotals, gt * 8 + (gt / SUPER + 1) * 8 + 16)) || (rc = ensure_dev(ctx, off, (n + 1) * 8 + 16)))
        return rc;
    if (!n) {
        if ((rc = ensure_dev(ctx, bytes, 16)))
            return rc;
        CK(cudaMemsetAsync(off.p, 0, 8, s));
        return REGK_OK;
    }
    MkGatherParams gp{};
    gp.n_dirs = n;
    gp.dir_len = len;
    gp.tile_total = (unsigned long long *)wk.gtotals.p;
    gp.super_total = gp.tile_total + gt;
    CK(cudaMemsetAsync(gp.super_total, 0, (gt / SUPER + 1) * 8, s));
    regk_mkdirp_len_kernel<<<(unsigned)gt, MK_TILE, 0, s>>>(gp);
    std::vector<unsigned long long> gs(gt / SUPER + 1);
    CK(cudaMemcpyAsync(gs.data(), gp.super_total, gs.size() * 8, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    for (unsigned long long v : gs)
        *total += v;
    if ((rc = ensure_dev(ctx, bytes, *total + 16)))
        return rc;
    WalkRebuildParams rp{};
    rp.n = n;
    rp.src0 = src0;
    rp.src1 = src1;
    rp.src_off = src_off;
    rp.sel = sel;
    rp.len = len;
    rp.tile_total = gp.tile_total;
    rp.super_total = gp.super_total;
    rp.out = (uint8_t *)bytes.p;
    rp.out_off = (unsigned long long *)off.p;
    regk_walk_rebuild_kernel<<<(unsigned)gt, MK_TILE, 0, s>>>(rp);
    CK(cudaGetLastError());
    *launches += 2;
    return REGK_OK;
}

/* The snapshot without its removed nodes, in order, their marks, versions and owners moving with them; a node marked
   replaced takes its data from `ds` (a refresh level's reply stream).  The pending count is recounted, the removed count
   is 0, and the path table is stale. */
static int walk_rebuild(regk_ctx *ctx, const uint8_t *ds, uint32_t *launches, const char *who)
{
    regk_ctx::Walk &wk = ctx->wk;
    cudaStream_t s = ctx->stream;
    const uint64_t m = wk.m;
    const uint64_t tiles = (m + RP_TILE - 1) / RP_TILE;
    const size_t tb = align16(tiles * 4) + (tiles / SUPER + 1) * 8;
    int rc;
    if ((rc = walk_rebuild_reserve(ctx, 0)))
        return rc;
    unsigned long long kc[2] = {0, 0};
    CK(cudaMemsetAsync(wk.kcount.p, 0, 16, s));
    WalkKeepParams kp{};
    kp.m = m;
    kp.mark = (const uint32_t *)wk.wmark.p;
    kp.path_off = (const unsigned long long *)wk.snap_off[0].p;
    kp.json_off = (const unsigned long long *)wk.snap_off[1].p;
    kp.ver = (const int32_t *)wk.ver.p;
    kp.own = (const long long *)wk.own.p;
    kp.rpos = (const unsigned long long *)wk.rpos.p;
    kp.rlen = (const uint32_t *)wk.rlen.p;
    kp.tile_total = (uint32_t *)wk.ktotals.p;
    kp.super_total = (unsigned long long *)((uint8_t *)wk.ktotals.p + align16(tiles * 4));
    kp.counters = (unsigned long long *)wk.kcount.p;
    kp.psrc = (unsigned long long *)wk.psrc.p;
    kp.dsrc = (unsigned long long *)wk.dsrc.p;
    kp.plen = (uint32_t *)wk.kplen.p;
    kp.dlen = (uint32_t *)wk.kdlen.p;
    kp.dsel = (uint8_t *)wk.dsel.p;
    kp.nmark = (uint32_t *)wk.wmark2.p;
    kp.nver = (int32_t *)wk.ver2.p;
    kp.nown = (long long *)wk.own2.p;
    if (m) {
        CK(cudaMemsetAsync(wk.ktotals.p, 0, tb, s));
        regk_walk_keep_count_kernel<<<(unsigned)tiles, RP_TILE, 0, s>>>(kp);
        regk_walk_keep_kernel<<<(unsigned)tiles, RP_TILE, 0, s>>>(kp);
        /* the armed bytes move with their nodes; not counted in `launches` (bookkeeping for regk_walk_setwatches) */
        regk_walk_keep_armed_kernel<<<(unsigned)tiles, RP_TILE, 0, s>>>(kp, (const uint8_t *)wk.armed.p, (uint8_t *)wk.armed2.p);
        /* so do the identities, a replaced node's only while its data bytes stay the same (regk_walk_resolve's
           bookkeeping, not counted either) */
        regk_walk_keep_ident_kernel<<<(unsigned)tiles, RP_TILE, 0, s>>>(kp, (const uint32_t *)wk.ident.p, (uint32_t *)wk.ident2.p,
            (const uint8_t *)wk.snap_bytes[1].p, ds);
        CK(cudaGetLastError());
        *launches += 2;
        CK(cudaMemcpyAsync(kc, kp.counters, 16, cudaMemcpyDeviceToHost, s));
        if ((rc = sync_or_fail(ctx, s, who)))
            return rc;
    }
    const uint64_t k = kc[0];
    uint64_t tot[2] = {0, 0};
    for (int g = 0; g < 2; g++)
        if ((rc = walk_pack(ctx, k, (const uint8_t *)wk.snap_bytes[g].p, g ? ds : nullptr, g ? kp.dsrc : kp.psrc,
                 g ? kp.dsel : nullptr, g ? kp.dlen : kp.plen, wk.snap2_bytes[g], wk.snap2_off[g], &tot[g], launches)))
            return rc;
    for (int g = 0; g < 2; g++) {
        std::swap(wk.snap_bytes[g], wk.snap2_bytes[g]);
        std::swap(wk.snap_off[g], wk.snap2_off[g]);
    }
    std::swap(wk.wmark, wk.wmark2);
    std::swap(wk.armed, wk.armed2);
    std::swap(wk.ident, wk.ident2);
    std::swap(wk.ver, wk.ver2);
    std::swap(wk.own, wk.own2);
    const unsigned long long mc[WM_NCOUNTERS] = {kc[1], 0ull};
    CK(cudaMemcpyAsync(wk.mcount.p, mc, sizeof mc, cudaMemcpyHostToDevice, s));
    CK(cudaStreamSynchronize(s));
    wk.sgen++;
    wk.m = k;
    wk.path_total = tot[0];
    wk.data_total = tot[1];
    wk.n_pending = kc[1];
    wk.n_removed = 0;
    wk.rgen++;
    return REGK_OK;
}

static int walk_append(regk_ctx *ctx, const uint8_t *ds, const uint8_t *fbytes, const unsigned long long *foff,
    const unsigned long long *data_pos, const WalkFoundParams &fp, uint64_t mf, uint32_t *launches);
static int walk_out(regk_ctx *ctx, const unsigned long long *hw, uint64_t ne, uint64_t n_listed, uint64_t n_list_missing,
    uint64_t n_list_error, uint64_t n_skipped, uint64_t consumed, uint32_t flags, uint32_t launches, float ms, regk_walk *out);

int regk_walk_start(regk_ctx *ctx, const uint8_t *roots, const uint64_t *root_off, uint64_t n_roots, uint32_t flags)
{
    if (!ctx || !root_off || (!roots && n_roots))
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_walk_start: NULL argument");
    if (flags)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_walk_start: flags must be 0 (the roots are host memory)");
    if (!n_roots)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_walk_start: no roots");
    for (uint64_t i = 0; i < n_roots; i++)
        if (root_off[i + 1] < root_off[i] || root_off[i + 1] - root_off[i] >= (1ull << 31))
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_walk_start: root %llu: offsets not monotone, or a root of 2^31 bytes "
                                                   "or more", (unsigned long long)i);
    std::vector<std::string> r(n_roots);
    std::map<std::string, uint64_t> first;
    for (uint64_t i = 0; i < n_roots; i++) {
        r[i].assign((const char *)roots + root_off[i], root_off[i + 1] - root_off[i]);
        first.emplace(r[i], i);
    }
    for (uint64_t i = 0; i < n_roots; i++) {
        const std::string &s = r[i];
        const uint32_t c = mkdir_components((const uint8_t *)s.data(), (uint32_t)s.size());
        if (s.empty() || c == MKDIR_INVALID)
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_walk_start: root %llu is a path ZooKeeper rejects",
                (unsigned long long)i);
        if (c == 0)
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_walk_start: root %llu is \"/\": its listing holds /zookeeper, and "
                                                   "'/' + name would give \"//name\"", (unsigned long long)i);
        const uint64_t j = first[s];
        if (j != i)
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_walk_start: root %llu equals root %llu", (unsigned long long)i,
                (unsigned long long)j);
        for (size_t t = 1; t < s.size(); t++) {
            auto a = s[t] == '/' ? first.find(s.substr(0, t)) : first.end();
            if (a != first.end())
                return fail(ctx, REGK_ERR_INVALID_ARG, "regk_walk_start: root %llu lies under root %llu", (unsigned long long)i,
                    (unsigned long long)a->second);
        }
    }
    CK(cudaSetDevice(ctx->device));
    regk_ctx::Walk &wk = ctx->wk;
    wk.active = wk.framed = false;              /* the earlier walk is gone even if staging fails */
    wk.sgen++;
    ctx->wr.have = false;                       /* regk_walk_resolve's kept text goes with the earlier walk */
    std::vector<uint8_t> pb;
    std::vector<unsigned long long> po(n_roots + 1, 0);
    std::vector<uint32_t> pl(n_roots);
    for (uint64_t i = 0; i < n_roots; i++) {
        pb.insert(pb.end(), r[i].begin(), r[i].end());
        po[i + 1] = pb.size();
        pl[i] = (uint32_t)r[i].size();
    }
    cudaStream_t s = ctx->stream;
    int rc;
    if ((rc = stage_in(ctx, wk.fbytes[0], pb.data(), pb.size(), s)) || (rc = stage_in(ctx, wk.foff[0], po.data(), po.size() * 8, s)) ||
        (rc = stage_in(ctx, wk.flen[0], pl.data(), pl.size() * 4, s)) || (rc = ensure_dev(ctx, wk.mcount, WM_NCOUNTERS * 8)))
        return rc;
    CK(cudaMemsetAsync(wk.mcount.p, 0, WM_NCOUNTERS * 8, s));
    if ((rc = sync_or_fail(ctx, s, "regk_walk_start")))
        return rc;
    wk.cur = 0;
    wk.f = n_roots;
    wk.fpt = pb.size();
    wk.m = wk.path_total = wk.data_total = 0;
    wk.level_off.assign(1, 0);
    /* the marks, the table and the refresh state go with the earlier walk */
    wk.watched = true;
    wk.framed_watch = wk.refreshed = wk.rlevel = wk.tab_valid = false;
    wk.n_pending = wk.n_removed = 0;
    wk.zxid = 0;
    wk.gate = false;
    wk.rgen++;
    wk.active = true;
    return REGK_OK;
}

int regk_walk_requests(regk_ctx *ctx, int32_t xid_base, uint32_t flags, regk_frames *out)
{
    if (!ctx || !out)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_walk_requests: NULL argument");
    memset(out, 0, sizeof *out);
    regk_ctx::Walk &wk = ctx->wk;
    if (flags & ~(REGK_OUT_DEVICE | REGK_ZK_WATCH))
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_walk_requests: unknown flags 0x%x", flags);
    if (!wk.active)
        return fail(ctx, REGK_ERR_STATE, "regk_walk_requests: no walk on this context; call regk_walk_start first");
    if (!wk.f)
        return fail(ctx, REGK_ERR_STATE, "regk_walk_requests: the walk is complete (its frontier is empty)");
    const uint64_t f = wk.f;
    if (f >= (1ull << 30))
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_walk_requests: a frontier of %llu nodes: must be below 2^30",
            (unsigned long long)f);
    for (int32_t reserved : {-1, -2})
        if ((uint64_t)((uint32_t)reserved - (uint32_t)xid_base) < 2 * f)
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_walk_requests: the xids [%d, %d + %llu) cover %d, which ZooKeeper uses "
                                                   "for %s", xid_base, xid_base, (unsigned long long)(2 * f), reserved,
                        reserved == -1 ? "watch notifications" : "pings");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    int rc;
    for (Event &ev : wk.ev)
        if ((rc = ensure_event(ctx, ev)))
            return rc;
    const unsigned long long sec1 = 17ull * f + wk.fpt, total = 2 * sec1;
    FrameBufs &fb = wk.frames;
    if ((rc = ensure_dev(ctx, fb.bytes, total + 16)) || (rc = ensure_dev(ctx, fb.off, (2 * f + 1) * 8)))
        return rc;
    WalkFrameParams p{};
    p.f = f;
    p.path_bytes = (const uint8_t *)wk.fbytes[wk.cur].p;
    p.path_off = (const unsigned long long *)wk.foff[wk.cur].p;
    p.xid_base = xid_base;
    p.sec1 = sec1;
    p.out = (uint8_t *)fb.bytes.p;
    p.out_off = (unsigned long long *)fb.off.p;
    CK(cudaEventRecord(wk.ev[0], s));
    regk_walk_frame_kernel<<<(unsigned)(2 * ((f + MK_TILE - 1) / MK_TILE)), MK_TILE, 0, s>>>(p);
    const bool watch = flags & REGK_ZK_WATCH;
    if (watch)
        regk_walk_watch_byte_kernel<<<(unsigned)((2 * f + 255) / 256), 256, 0, s>>>(p.out, p.out_off, 2 * f);
    CK(cudaGetLastError());
    CK(cudaEventRecord(wk.ev[1], s));
    const void *bytes = fb.bytes.p, *off = fb.off.p;
    if (!(flags & REGK_OUT_DEVICE)) {
        if ((rc = to_host(ctx, fb.h_bytes, fb.bytes.p, total, s)) || (rc = to_host(ctx, fb.h_off, fb.off.p, (2 * f + 1) * 8, s)))
            return rc;
        bytes = fb.h_bytes.p;
        off = fb.h_off.p;
    }
    if ((rc = sync_or_fail(ctx, s, "regk_walk_requests")))
        return rc;
    float ms = 0;
    cudaEventElapsedTime(&ms, wk.ev[0], wk.ev[1]);
    wk.framed = true;
    wk.framed_watch = watch;
    wk.xid = xid_base;
    out->n = 2 * f;
    out->total = total;
    out->flags = flags & REGK_OUT_DEVICE;
    out->launches = watch ? 2 : 1;
    out->frame_bytes = (const uint8_t *)bytes;
    out->frame_off = (const uint64_t *)off;
    out->kernel_ms = ms;
    return REGK_OK;
}

int regk_read_walk(regk_ctx *ctx, const uint8_t *bytes, uint64_t len, uint32_t flags, regk_walk *out)
{
    const char *who = "regk_read_walk";
    if (!ctx || !out)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_walk: NULL argument");
    memset(out, 0, sizeof *out);
    regk_ctx::Walk &wk = ctx->wk;
    if (flags & ~(REGK_IN_DEVICE | REGK_OUT_DEVICE))
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_walk: unknown flags 0x%x", flags);
    if (!wk.active || !wk.framed)
        return fail(ctx, REGK_ERR_STATE, "regk_read_walk: no framing of the walk's current frontier (regk_walk_requests)");
    if (!bytes && len)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_walk: NULL stream of %llu bytes", (unsigned long long)len);
    const bool in_dev = flags & REGK_IN_DEVICE;
    if (in_dev && ((uintptr_t)bytes & 15u))
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_walk: misaligned device stream (16-byte alignment needed)");
    const uint64_t f = wk.f;
    const int32_t xb = wk.xid, xc = (int32_t)((uint32_t)xb + (uint32_t)f);
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    int rc;
    for (Event &ev : wk.ev)
        if ((rc = ensure_event(ctx, ev)))
            return rc;
    const uint8_t *ds = bytes;
    if (!in_dev) {
        if ((rc = stage_in(ctx, wk.stream, bytes, len, s)))
            return rc;
        ds = (const uint8_t *)wk.stream.p;
    }
    const int cur = wk.cur, nx = 1 - cur;
    const uint8_t *fbytes = (const uint8_t *)wk.fbytes[cur].p;
    const unsigned long long *foff = (const unsigned long long *)wk.foff[cur].p;
    const uint64_t nblk = (len + 15) / 16, tiles_s = (nblk + RP_TILE - 1) / RP_TILE;
    const size_t totals_bytes = align16(tiles_s * 4) + (tiles_s / SUPER + 1) * 8;
    const size_t f8 = f * 8 + 16, f4 = f * 4 + 16;
    if ((rc = ensure_dev(ctx, wk.word, nblk * 4 + 16)) || (rc = ensure_dev(ctx, wk.totals, totals_bytes)) ||
        (rc = ensure_dev(ctx, wk.tile_base, tiles_s * 8 + 16)) || (rc = ensure_dev(ctx, wk.err, f4)) ||
        (rc = ensure_dev(ctx, wk.data_pos, f8)) || (rc = ensure_dev(ctx, wk.dlen, f4)) || (rc = ensure_dev(ctx, wk.dver, f4)) ||
        (rc = ensure_dev(ctx, wk.down, f8)) || (rc = ensure_dev(ctx, wk.count, CQ_NCOUNTERS * 8)) ||
        (rc = ensure_host(ctx, wk.h_count, CQ_NCOUNTERS * 8)) || (rc = ensure_dev(ctx, wk.zmax, 16)))
        return rc;
    unsigned long long *hc = (unsigned long long *)wk.h_count.p;
    /* 1. the getData section: the frame chain from 0, the replies of the f nodes (regk_replies.cuh) */
    RepParams p{};
    p.s = ds;
    p.len = len;
    p.xid_base = xb;
    p.n = f;
    p.word = (uint32_t *)wk.word.p;
    p.tile_total = (uint32_t *)wk.totals.p;
    p.super_total = (unsigned long long *)((uint8_t *)wk.totals.p + align16(tiles_s * 4));
    p.tile_base = (unsigned long long *)wk.tile_base.p;
    p.err = (int32_t *)wk.err.p;
    p.data_pos = (unsigned long long *)wk.data_pos.p;
    p.dlen = (uint32_t *)wk.dlen.p;
    p.ver = (int32_t *)wk.dver.p;
    p.own = (long long *)wk.down.p;
    p.counters = (unsigned long long *)wk.count.p;
    CK(cudaMemsetAsync(p.counters, 0, CQ_NCOUNTERS * 8, s));
    CK(cudaMemsetAsync(p.counters + RQ_ERR, 0xFF, 8, s));
    CK(cudaMemsetAsync(p.tile_total, 0, totals_bytes, s));
    CK(cudaEventRecord(wk.ev[0], s));
    uint32_t launches = 0;
    if (len) {
        regk_replies_cand_kernel<<<(unsigned)tiles_s, RP_TILE, 0, s>>>(p);
        CK(cudaGetLastError());
        launches++;
    }
    RepParams pg = p;
    uint32_t *J = nullptr;
    if ((rc = chain_pass(ctx, &pg, tiles_s, ~0ull, wk.cand, wk.mark, wk.jump, [&](const RepParams &q) {
            regk_children_seed_kernel<<<1, 256, 0, s>>>(q, nullptr, nullptr, 1, 0ull);
        }, &J, &launches, who)))
        return rc;
    if (pg.C) {
        const uint64_t tiles_c = (pg.C + RP_TILE - 1) / RP_TILE;
        const size_t t2 = align16(tiles_c * 4) + (tiles_c / SUPER + 1) * 8;
        if ((rc = ensure_dev(ctx, wk.totals2, t2)))
            return rc;
        RepParams p2 = pg;
        p2.tile_total = (uint32_t *)wk.totals2.p;
        p2.super_total = (unsigned long long *)((uint8_t *)wk.totals2.p + align16(tiles_c * 4));
        CK(cudaMemsetAsync(wk.totals2.p, 0, t2, s));
        regk_replies_chain_count_kernel<<<(unsigned)tiles_c, RP_TILE, 0, s>>>(p2);
        regk_replies_chain_kernel<<<(unsigned)tiles_c, RP_TILE, 0, s>>>(p2);
        CK(cudaGetLastError());
        launches += 2;
    }
    CK(cudaMemcpyAsync(hc, p.counters, CQ_NCOUNTERS * 8, cudaMemcpyDeviceToHost, s));
    if ((rc = sync_or_fail(ctx, s, who)))
        return rc;
    if (hc[RQ_ERR] != ~0ull) {
        const uint64_t k = hc[RQ_ERR] >> 8;
        const uint32_t code = (uint32_t)(hc[RQ_ERR] & 0xFF);
        unsigned long long dpos = 0;
        CK(cudaMemcpyAsync(&dpos, p.data_pos + k, 8, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_walk: byte %llu: %s; expected the getData reply to node %llu (xid %d)",
            dpos - 24, reply_reason(code), (unsigned long long)k, (int32_t)((uint32_t)xb + (uint32_t)k));
    }
    if (hc[RQ_NREP] < f) {
        uint64_t stop = 0;
        if (pg.C) {
            regk_replies_stop_kernel<<<(unsigned)((pg.C + 255) / 256), 256, 0, s>>>(pg);
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
        const uint32_t code = reply_head(head, avail, xb, f, &h);
        const int32_t want = (int32_t)((uint32_t)xb + (uint32_t)done);
        if (code == RP_TRUNC)
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_walk: byte %llu: the stream ends before the getData reply to node "
                                                   "%llu (xid %d) is complete; %llu of %llu replies complete",
                        (unsigned long long)stop, (unsigned long long)done, want, (unsigned long long)done, (unsigned long long)f);
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_walk: byte %llu: %s (len %d, xid %d); expected the getData reply to "
                                               "node %llu (xid %d)", (unsigned long long)stop,
                    code ? reply_reason(code) : "internal error", h.len, h.xid, (unsigned long long)done, want);
    }
    const uint64_t start = hc[RQ_CONSUMED], gd_skipped = hc[RQ_SKIP];
    /* 2. the getChildren section from the getData section's end (regk_children.cuh), the listing's entries */
    if ((rc = ensure_dev(ctx, wk.cword, nblk * 4 + 16)) || (rc = ensure_dev(ctx, wk.ctotals, totals_bytes)) ||
        (rc = ensure_dev(ctx, wk.ctile_base, tiles_s * 8 + 16)) || (rc = ensure_dev(ctx, wk.fpos, f8)) ||
        (rc = ensure_dev(ctx, wk.fend, f8)) || (rc = ensure_dev(ctx, wk.cerr, f4)) || (rc = ensure_dev(ctx, wk.cnt, f4)) ||
        (rc = ensure_dev(ctx, wk.seed_g, f4)) || (rc = ensure_dev(ctx, wk.last_g1, f4)) ||
        (rc = ensure_dev(ctx, wk.name_bad, f4)) || (rc = ensure_dev(ctx, wk.end_pos, f8)) ||
        (rc = ensure_dev(ctx, wk.fault_pos, f8)) || (rc = ensure_dev(ctx, wk.child_off, f8)))
        return rc;
    ChParams cp{};
    RepParams &pc = cp.r;
    pc.s = ds;
    pc.len = len;
    pc.xid_base = xc;
    pc.n = f;
    pc.word = (uint32_t *)wk.cword.p;
    pc.tile_total = (uint32_t *)wk.ctotals.p;
    pc.super_total = (unsigned long long *)((uint8_t *)wk.ctotals.p + align16(tiles_s * 4));
    pc.tile_base = (unsigned long long *)wk.ctile_base.p;
    pc.counters = p.counters;
    cp.start = start;
    cp.d = f;
    cp.fpos = (unsigned long long *)wk.fpos.p;
    cp.fend = (unsigned long long *)wk.fend.p;
    cp.err = (int32_t *)wk.cerr.p;
    cp.cnt = (uint32_t *)wk.cnt.p;
    cp.seed_g = (uint32_t *)wk.seed_g.p;
    cp.last_g1 = (uint32_t *)wk.last_g1.p;
    cp.name_bad = (uint32_t *)wk.name_bad.p;
    cp.end_pos = (unsigned long long *)wk.end_pos.p;
    cp.fault_pos = (unsigned long long *)wk.fault_pos.p;
    cp.child_off = (unsigned long long *)wk.child_off.p;
    cp.dir_len = (const uint32_t *)wk.flen[cur].p;
    const RepParams pc0 = pc;
    CK(cudaMemsetAsync(p.counters, 0, CQ_NCOUNTERS * 8, s));
    CK(cudaMemsetAsync(p.counters + RQ_ERR, 0xFF, 8, s));
    CK(cudaMemsetAsync(p.counters + CQ_ENT_ERR, 0xFF, 8, s));
    CK(cudaMemsetAsync(pc.tile_total, 0, totals_bytes, s));
    RepParams pf = pc;
    if (len) {
        regk_children_cand_kernel<<<(unsigned)tiles_s, RP_TILE, 0, s>>>(cp);
        CK(cudaGetLastError());
        launches++;
        if ((rc = chain_pass(ctx, &pf, tiles_s, ~0ull, wk.ccand, wk.cmark, wk.cjump, [&](const RepParams &q) {
                regk_children_seed_kernel<<<1, 256, 0, s>>>(q, nullptr, nullptr, 1, start);
            }, &J, &launches, who)))
            return rc;
        if (pf.C) {
            const uint64_t tiles_c = (pf.C + RP_TILE - 1) / RP_TILE;
            const size_t t2 = align16(tiles_c * 4) + (tiles_c / SUPER + 1) * 8;
            if ((rc = ensure_dev(ctx, wk.ctotals2, t2)))
                return rc;
            cp.r = pf;
            cp.r.tile_total = (uint32_t *)wk.ctotals2.p;
            cp.r.super_total = (unsigned long long *)((uint8_t *)wk.ctotals2.p + align16(tiles_c * 4));
            CK(cudaMemsetAsync(wk.ctotals2.p, 0, t2, s));
            regk_replies_chain_count_kernel<<<(unsigned)tiles_c, RP_TILE, 0, s>>>(cp.r);
            regk_children_chain_kernel<<<(unsigned)tiles_c, RP_TILE, 0, s>>>(cp);
            CK(cudaGetLastError());
            launches += 2;
        }
    }
    CK(cudaMemcpyAsync(hc, p.counters, CQ_NCOUNTERS * 8, cudaMemcpyDeviceToHost, s));
    if ((rc = sync_or_fail(ctx, s, who)))
        return rc;
    const uint64_t frame_err_k = hc[RQ_ERR] != ~0ull ? hc[RQ_ERR] >> 8 : f;
    const uint64_t d_eff = std::min<uint64_t>(std::min<uint64_t>(frame_err_k, hc[RQ_NREP]), f);
    const uint64_t ch_skipped = hc[RQ_SKIP], n_listed = hc[RQ_FOUND], n_list_missing = hc[RQ_MISSING];
    const uint64_t n_list_error = hc[RQ_ERROR], consumed = hc[RQ_CONSUMED];
    uint64_t ne = 0, Ce = 0;
    if (d_eff) {
        cp.d_eff = d_eff;
        if ((rc = ensure_dev(ctx, wk.eword, nblk * 4 + 16)) || (rc = ensure_dev(ctx, wk.etotals, totals_bytes)) ||
            (rc = ensure_dev(ctx, wk.etile_base, tiles_s * 8 + 16)))
            return rc;
        RepParams pe = pc0;
        pe.word = (uint32_t *)wk.eword.p;
        pe.tile_total = (uint32_t *)wk.etotals.p;
        pe.super_total = (unsigned long long *)((uint8_t *)wk.etotals.p + align16(tiles_s * 4));
        pe.tile_base = (unsigned long long *)wk.etile_base.p;
        CK(cudaMemsetAsync(pe.tile_total, 0, totals_bytes, s));
        CK(cudaMemsetAsync(cp.seed_g, 0xFF, d_eff * 4, s));
        CK(cudaMemsetAsync(cp.name_bad, 0xFF, d_eff * 4, s));
        CK(cudaMemsetAsync(cp.last_g1, 0, d_eff * 4, s));
        cp.r = pe;
        regk_children_ent_cand_kernel<<<(unsigned)tiles_s, RP_TILE, 0, s>>>(cp);
        CK(cudaGetLastError());
        launches++;
        const unsigned gd = (unsigned)((d_eff + 255) / 256);
        if ((rc = chain_pass(ctx, &pe, tiles_s, hc[CQ_MAXC] + 1, wk.ecand, wk.emark, wk.ejump, [&](const RepParams &q) {
                regk_children_seed_kernel<<<gd, 256, 0, s>>>(q, cp.fpos, cp.cnt, d_eff, 24ull);
            }, &J, &launches, who)))
            return rc;
        Ce = pe.C;
        /* the entries' listing path lengths go straight to the next frontier's lengths */
        if ((rc = ensure_dev(ctx, wk.ent_pos, Ce * 8 + 16)) || (rc = ensure_dev(ctx, wk.ent_nlen, Ce * 4 + 16)) ||
            (rc = ensure_dev(ctx, wk.ent_k, Ce * 4 + 16)) || (rc = ensure_dev(ctx, wk.flen[nx], Ce * 4 + 16)))
            return rc;
        cp.j0 = J;
        cp.ent_pos = (unsigned long long *)wk.ent_pos.p;
        cp.ent_nlen = (uint32_t *)wk.ent_nlen.p;
        cp.ent_k = (uint32_t *)wk.ent_k.p;
        cp.ent_plen = (uint32_t *)wk.flen[nx].p;
        cp.r = pe;
        if (Ce) {
            const uint64_t tiles_e = (Ce + RP_TILE - 1) / RP_TILE;
            const size_t t2 = align16(tiles_e * 4) + (tiles_e / SUPER + 1) * 8;
            if ((rc = ensure_dev(ctx, wk.etotals2, t2)))
                return rc;
            cp.r.tile_total = (uint32_t *)wk.etotals2.p;
            cp.r.super_total = (unsigned long long *)((uint8_t *)wk.etotals2.p + align16(tiles_e * 4));
            CK(cudaMemsetAsync(wk.etotals2.p, 0, t2, s));
            regk_children_ent_count_kernel<<<(unsigned)tiles_e, RP_TILE, 0, s>>>(cp.r);
            regk_children_ent_kernel<<<(unsigned)tiles_e, RP_TILE, 0, s>>>(cp);
            launches += 2;
        }
        regk_children_ent_frame_kernel<<<gd, 256, 0, s>>>(cp);
        CK(cudaGetLastError());
        launches++;
        CK(cudaMemcpyAsync(hc, p.counters, CQ_NCOUNTERS * 8, cudaMemcpyDeviceToHost, s));
        if ((rc = sync_or_fail(ctx, s, who)))
            return rc;
        ne = hc[CQ_NENT];
    }
    if (hc[CQ_ENT_ERR] != ~0ull) {
        const uint64_t k = hc[CQ_ENT_ERR] >> 8;
        const uint32_t code = (uint32_t)(hc[CQ_ENT_ERR] & 0xFF);
        unsigned long long at[2] = {0, 0};
        CK(cudaMemcpyAsync(&at[0], cp.fault_pos + k, 8, cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(&at[1], cp.fpos + k, 8, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_walk: byte %llu: %s (entry of the reply frame at byte %llu); expected "
                                               "the getChildren reply to node %llu (xid %d)", at[0], children_reason(code), at[1],
                    (unsigned long long)k, (int32_t)((uint32_t)xc + (uint32_t)k));
    }
    if (hc[RQ_ERR] != ~0ull) {
        const uint64_t k = hc[RQ_ERR] >> 8;
        const uint32_t code = (uint32_t)(hc[RQ_ERR] & 0xFF);
        unsigned long long pos = 0;
        CK(cudaMemcpyAsync(&pos, cp.fpos + k, 8, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_walk: byte %llu: %s; expected the getChildren reply to node %llu "
                                               "(xid %d)", pos, children_reason(code), (unsigned long long)k,
                    (int32_t)((uint32_t)xc + (uint32_t)k));
    }
    if (hc[RQ_NREP] < f) {
        uint64_t stop = start;
        if (pf.C) {
            regk_replies_stop_kernel<<<(unsigned)((pf.C + 255) / 256), 256, 0, s>>>(pf);
            CK(cudaGetLastError());
            CK(cudaMemcpyAsync(hc + RQ_STOP, p.counters + RQ_STOP, 8, cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
            stop = std::max<uint64_t>(stop, hc[RQ_STOP]);
        }
        const uint64_t done = hc[RQ_NREP];
        uint8_t head[24] = {0};
        const uint64_t avail = len - stop, take = std::min<uint64_t>(avail, sizeof head);
        if (take) {
            CK(cudaMemcpyAsync(head, ds + stop, take, cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
        }
        ChildHead h;
        const uint32_t code = children_head(head, avail, xc, f, &h);
        const int32_t want = (int32_t)((uint32_t)xc + (uint32_t)done);
        if (code == CH_TRUNC)
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_walk: byte %llu: the stream ends before the getChildren reply to "
                                                   "node %llu (xid %d) is complete; %llu of %llu replies complete",
                        (unsigned long long)stop, (unsigned long long)done, want, (unsigned long long)done, (unsigned long long)f);
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_walk: byte %llu: %s (len %d, xid %d); expected the getChildren reply "
                                               "to node %llu (xid %d)", (unsigned long long)stop,
                    code ? children_reason(code) : "internal error", h.len, h.xid, (unsigned long long)done, want);
    }
    if (ne >= 0xFFFFFFFFull)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_read_walk: %llu children: must be below 2^32 - 1", (unsigned long long)ne);
    /* 3. the next frontier: listing path e = frontier path + '/' + name, packed from 0 */
    uint64_t lst_total = 0;
    {
        const uint64_t gt = (ne + MK_TILE - 1) / MK_TILE;
        if ((rc = ensure_dev(ctx, wk.gtotals, gt * 8 + (gt / SUPER + 1) * 8 + 16)) ||
            (rc = ensure_dev(ctx, wk.foff[nx], (ne + 1) * 8)) || (rc = ensure_dev(ctx, wk.flen[nx], ne * 4 + 16)))
            return rc;
        if (ne) {
            MkGatherParams gp{};
            gp.n_dirs = ne;
            gp.dir_len = cp.ent_plen;
            gp.tile_total = (unsigned long long *)wk.gtotals.p;
            gp.super_total = gp.tile_total + gt;
            CK(cudaMemsetAsync(gp.super_total, 0, (gt / SUPER + 1) * 8, s));
            regk_mkdirp_len_kernel<<<(unsigned)gt, MK_TILE, 0, s>>>(gp);
            std::vector<unsigned long long> gs(gt / SUPER + 1);
            CK(cudaMemcpyAsync(gs.data(), gp.super_total, gs.size() * 8, cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
            for (unsigned long long v : gs)
                lst_total += v;
            if ((rc = ensure_dev(ctx, wk.fbytes[nx], lst_total + 16)))
                return rc;
            ChGatherParams g{};
            g.n = ne;
            g.tile_total = gp.tile_total;
            g.super_total = gp.super_total;
            g.ent_k = cp.ent_k;
            g.ent_nlen = cp.ent_nlen;
            g.ent_plen = cp.ent_plen;
            g.ent_pos = cp.ent_pos;
            g.dir_bytes = fbytes;
            g.dir_off = foff;
            g.s = ds;
            g.out_bytes = (uint8_t *)wk.fbytes[nx].p;
            g.out_off = (unsigned long long *)wk.foff[nx].p;
            regk_children_gather_kernel<<<(unsigned)gt, MK_TILE, 0, s>>>(g);
            CK(cudaGetLastError());
            launches += 2;
        } else {
            if ((rc = ensure_dev(ctx, wk.fbytes[nx], 16)))
                return rc;
            CK(cudaMemsetAsync(wk.foff[nx].p, 0, 8, s));
        }
    }
    /* 3b. watches: a refresh level's getData replies land on their nodes (regk_walk_refresh), and once a walk has been
       refreshed every listing drops the paths the snapshot already holds */
    uint64_t nf = ne;
    if (wk.rlevel) {
        /* the table and every buffer the filter and the rebuild need come first: once the replies are applied, nothing
           that follows can fail on an allocation */
        uint64_t built;
        if ((rc = walk_table(ctx, &built, &launches, who)) || (rc = walk_filter_reserve(ctx, ne, lst_total)) ||
            (rc = walk_rebuild_reserve(ctx, len)))
            return rc;
        WalkApplyParams ap{};
        ap.f = f;
        ap.fnode = (const unsigned long long *)wk.fnode.p;
        ap.err = p.err;
        ap.ver = p.ver;
        ap.own = p.own;
        ap.data_pos = p.data_pos;
        ap.dlen = p.dlen;
        ap.mark = (uint32_t *)wk.wmark.p;
        ap.snap_ver = (int32_t *)wk.ver.p;
        ap.snap_own = (long long *)wk.own.p;
        ap.rpos = (unsigned long long *)wk.rpos.p;
        ap.rlen = (uint32_t *)wk.rlen.p;
        regk_walk_apply_kernel<<<(unsigned)((f + 255) / 256), 256, 0, s>>>(ap);
        /* the frontier nodes' armed bytes, before the rebuild renumbers them (not counted in `launches`) */
        WalkArmParams am{};
        am.n = f;
        am.fnode = ap.fnode;
        am.err = p.err;
        am.cerr = (const int32_t *)wk.cerr.p;
        am.watch = wk.framed_watch ? 1u : 0u;
        am.armed = (uint8_t *)wk.armed.p;
        regk_walk_arm_kernel<<<(unsigned)((f + 255) / 256), 256, 0, s>>>(am);
        CK(cudaGetLastError());
        launches++;
    }
    if (wk.refreshed && ne && (rc = walk_filter(ctx, nx, ne, wk.rlevel, &nf, &lst_total, &launches, who)))
        return rc;
    /* 4. the level's nodes: the found getData replies in frontier order, with their stats */
    const uint64_t tiles_r = (f + RP_TILE - 1) / RP_TILE;
    const size_t ft_bytes = align16(tiles_r * 4) + (tiles_r / SUPER + 1) * 8;
    if ((rc = ensure_dev(ctx, wk.ftotals, ft_bytes)) || (rc = ensure_dev(ctx, wk.node_rec, f8)) ||
        (rc = ensure_dev(ctx, wk.node_ver, f4)) || (rc = ensure_dev(ctx, wk.node_own, f8)) ||
        (rc = ensure_dev(ctx, wk.node_plen, f4)) || (rc = ensure_dev(ctx, wk.node_dlen, f4)) ||
        (rc = ensure_dev(ctx, wk.wcount, WK_NCOUNTERS * 8)) || (rc = ensure_host(ctx, wk.h_wcount, WK_NCOUNTERS * 8)))
        return rc;
    WalkFoundParams fp{};
    fp.f = f;
    fp.err = p.err;
    fp.dlen = p.dlen;
    fp.ver = p.ver;
    fp.own = p.own;
    fp.path_off = foff;
    fp.tile_total = (uint32_t *)wk.ftotals.p;
    fp.super_total = (unsigned long long *)((uint8_t *)wk.ftotals.p + align16(tiles_r * 4));
    fp.node_rec = (unsigned long long *)wk.node_rec.p;
    fp.node_ver = (int32_t *)wk.node_ver.p;
    fp.node_own = (long long *)wk.node_own.p;
    fp.node_plen = (uint32_t *)wk.node_plen.p;
    fp.node_dlen = (uint32_t *)wk.node_dlen.p;
    fp.counters = (unsigned long long *)wk.wcount.p;
    CK(cudaMemsetAsync(wk.ftotals.p, 0, ft_bytes, s));
    CK(cudaMemsetAsync(fp.counters, 0, WK_NCOUNTERS * 8, s));
    regk_walk_found_count_kernel<<<(unsigned)tiles_r, RP_TILE, 0, s>>>(fp);
    regk_walk_found_kernel<<<(unsigned)tiles_r, RP_TILE, 0, s>>>(fp);
    CK(cudaGetLastError());
    launches += 2;
    unsigned long long *hw = (unsigned long long *)wk.h_wcount.p;
    CK(cudaMemcpyAsync(hw, fp.counters, WK_NCOUNTERS * 8, cudaMemcpyDeviceToHost, s));
    if ((rc = sync_or_fail(ctx, s, who)))
        return rc;
    const uint64_t mf = hw[WK_FOUND], m0 = wk.m;
    if (wk.rlevel) {
        /* 5'. a refresh level appends nothing: the snapshot is rebuilt without its removed nodes, with the replaced data */
        if ((rc = walk_rebuild(ctx, ds, &launches, who)))
            return rc;
    } else if ((rc = walk_append(ctx, ds, fbytes, foff, p.data_pos, fp, mf, &launches)))
        return rc;
    CK(cudaEventRecord(wk.ev[1], s));
    /* regk_walk_setwatches' bookkeeping, outside the read's launches and kernel_ms: the appended nodes' armed bytes,
       and the largest zxid of both sections' reply frames */
    if (!wk.rlevel && mf) {
        WalkArmParams am{};
        am.n = mf;
        am.node_rec = fp.node_rec;
        am.base = m0;
        am.err = p.err;
        am.cerr = (const int32_t *)wk.cerr.p;
        am.watch = wk.framed_watch ? 1u : 0u;
        am.armed = (uint8_t *)wk.armed.p;
        regk_walk_arm_kernel<<<(unsigned)((mf + 255) / 256), 256, 0, s>>>(am);
        /* regk_walk_resolve's: an appended node has no identity */
        CK(cudaMemsetAsync((uint32_t *)wk.ident.p + m0, 0xFF, mf * 4, s));
    }
    CK(cudaMemsetAsync(wk.zmax.p, 0, 8, s));
    for (const RepParams *q : {&pg, &pf})
        if (q->C)
            regk_events_zxid_kernel<<<(unsigned)((q->C + 255) / 256), 256, 0, s>>>(*q, (long long *)wk.zmax.p);
    CK(cudaGetLastError());
    long long zmax = 0;
    CK(cudaMemcpyAsync(&zmax, wk.zmax.p, 8, cudaMemcpyDeviceToHost, s));
    if ((rc = sync_or_fail(ctx, s, who)))
        return rc;
    wk.zxid = std::max(wk.zxid, zmax);
    float ms = 0;
    cudaEventElapsedTime(&ms, wk.ev[0], wk.ev[1]);
    /* the level is in: the listing is the next frontier, unframed */
    if (wk.rlevel)
        wk.level_off.assign(1, wk.m);
    else
        wk.level_off.push_back(wk.m);
    wk.watched = wk.watched && wk.framed_watch;
    wk.rlevel = false;
    wk.cur = nx;
    wk.f = nf;
    wk.fpt = lst_total;
    wk.framed = false;
    out->level = wk.level_off.size() - 1;
    out->m = wk.m;
    out->n_frontier = nf;
    return walk_out(ctx, hw, ne, n_listed, n_list_missing, n_list_error, gd_skipped + ch_skipped, consumed, flags, launches,
                    ms, out);
}

/* One plain level's found nodes appended to the snapshot: their paths (from the frontier) and data (from the stream)
   packed, then written at the snapshot streams' ends; version, owner and a clear mark per node. */
static int walk_append(regk_ctx *ctx, const uint8_t *ds, const uint8_t *fbytes, const unsigned long long *foff,
    const unsigned long long *data_pos, const WalkFoundParams &fp, uint64_t mf, uint32_t *launches)
{
    regk_ctx::Walk &wk = ctx->wk;
    cudaStream_t s = ctx->stream;
    const uint64_t m0 = wk.m;
    const void *was[4] = {wk.snap_bytes[0].p, wk.snap_bytes[1].p, wk.snap_off[0].p, wk.snap_off[1].p};
    int rc;
    uint64_t tot[2] = {0, 0};
    for (int g = 0; g < 2; g++) {
        uint32_t l = 0;
        if ((rc = pack_strings(ctx, mf, g ? ds : fbytes, g ? data_pos : foff, fp.node_rec, g ? fp.node_dlen : fp.node_plen,
                 wk.gtotals, wk.lvl_bytes[g], wk.lvl_off[g], &tot[g], &l)))
            return rc;
        *launches += l;
    }
    const uint64_t at[2] = {wk.path_total, wk.data_total};
    for (int g = 0; g < 2; g++)
        if ((rc = walk_grow(ctx, wk.snap_bytes[g], at[g], at[g] + tot[g] + 16)) ||
            (rc = walk_grow(ctx, wk.snap_off[g], m0 * 8, (m0 + mf + 1) * 8)))
            return rc;
    if ((rc = walk_grow(ctx, wk.ver, m0 * 4, (m0 + mf) * 4 + 16)) || (rc = walk_grow(ctx, wk.own, m0 * 8, (m0 + mf) * 8 + 16)) ||
        (rc = walk_grow(ctx, wk.wmark, m0 * 4, (m0 + mf) * 4 + 16)) || (rc = walk_grow(ctx, wk.armed, m0, m0 + mf + 16)) ||
        (rc = walk_grow(ctx, wk.ident, m0 * 4, (m0 + mf) * 4 + 16)))
        return rc;
    for (int g = 0; g < 2; g++) {
        WalkAppendParams ap{};
        ap.src = (const uint8_t *)wk.lvl_bytes[g].p;
        ap.len = tot[g];
        ap.dst = (uint8_t *)wk.snap_bytes[g].p;
        ap.at = at[g];
        ap.src_off = (const unsigned long long *)wk.lvl_off[g].p;
        ap.n = mf;
        ap.dst_off = (unsigned long long *)wk.snap_off[g].p + m0;
        const uint64_t nb = (at[g] + tot[g] - (at[g] & ~15ull) + 15) / 16, th = std::max<uint64_t>(nb, mf + 1);
        regk_walk_append_kernel<<<(unsigned)((th + 255) / 256), 256, 0, s>>>(ap);
        CK(cudaGetLastError());
        (*launches)++;
    }
    if (mf) {
        CK(cudaMemcpyAsync((int32_t *)wk.ver.p + m0, fp.node_ver, mf * 4, cudaMemcpyDeviceToDevice, s));
        CK(cudaMemcpyAsync((long long *)wk.own.p + m0, fp.node_own, mf * 8, cudaMemcpyDeviceToDevice, s));
        CK(cudaMemsetAsync((uint32_t *)wk.wmark.p + m0, 0, mf * 4, s));
    }
    if (mf || was[0] != wk.snap_bytes[0].p || was[1] != wk.snap_bytes[1].p || was[2] != wk.snap_off[0].p ||
        was[3] != wk.snap_off[1].p)
        wk.sgen++;
    wk.m = m0 + mf;
    wk.path_total += tot[0];
    wk.data_total += tot[1];
    return REGK_OK;
}

/* regk_read_walk's result: the level's counts and the walk's state */
static int walk_out(regk_ctx *ctx, const unsigned long long *hw, uint64_t ne, uint64_t n_listed, uint64_t n_list_missing,
    uint64_t n_list_error, uint64_t n_skipped, uint64_t consumed, uint32_t flags, uint32_t launches, float ms, regk_walk *out)
{
    regk_ctx::Walk &wk = ctx->wk;
    out->n_found = hw[WK_FOUND];
    out->n_missing = hw[WK_MISSING];
    out->n_error = hw[WK_ERROR];
    out->n_listed = n_listed;
    out->n_list_missing = n_list_missing;
    out->n_list_error = n_list_error;
    out->n_children = ne;
    out->n_skipped = n_skipped;
    out->consumed = consumed;
    out->flags = flags & REGK_OUT_DEVICE;
    out->launches = launches;
    out->level_off = wk.level_off.data();
    out->snapshot.n = wk.m;
    out->snapshot.flags = REGK_IN_DEVICE;
    out->snapshot.path_total = wk.path_total;
    out->snapshot.json_total = wk.data_total;
    out->snapshot.path_bytes = (const uint8_t *)wk.snap_bytes[0].p;
    out->snapshot.path_off = (const uint64_t *)wk.snap_off[0].p;
    out->snapshot.json_bytes = (const uint8_t *)wk.snap_bytes[1].p;
    out->snapshot.json_off = (const uint64_t *)wk.snap_off[1].p;
    out->version = (const int32_t *)wk.ver.p;
    out->ephemeral_owner = (const int64_t *)wk.own.p;
    out->kernel_ms = ms;
    return REGK_OK;
}

int regk_walk_events(regk_ctx *ctx, const uint8_t *bytes, uint64_t len, uint64_t start, const regk_events_opts *o,
    regk_walk_events_out *out)
{
    const char *who = "regk_walk_events";
    if (!ctx || !o || !out)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_walk_events: NULL argument");
    memset(out, 0, sizeof *out);
    regk_ctx::Walk &wk = ctx->wk;
    if (!wk.active)
        return fail(ctx, REGK_ERR_STATE, "regk_walk_events: no walk on this context; call regk_walk_start first");
    if (!wk.watched)
        return fail(ctx, REGK_ERR_STATE, "regk_walk_events: the walk is unwatched (a level was framed without "
                                         "REGK_ZK_WATCH); start a new walk with watches");
    if (o->flags & ~(REGK_IN_DEVICE | REGK_OUT_DEVICE))
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_walk_events: unknown flags 0x%x", o->flags);
    if (!bytes && len)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_walk_events: NULL stream of %llu bytes", (unsigned long long)len);
    if (start > len)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_walk_events: start %llu is past the stream's %llu bytes",
            (unsigned long long)start, (unsigned long long)len);
    const bool in_dev = o->flags & REGK_IN_DEVICE, dev_out = o->flags & REGK_OUT_DEVICE;
    if (in_dev && ((uintptr_t)bytes & 15u))
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_walk_events: misaligned device stream (16-byte alignment needed)");
    const int32_t xb = o->xid_base;
    const uint64_t nx = o->n_xids;
    for (int32_t reserved : {-1, -2})
        if ((uint64_t)((uint32_t)reserved - (uint32_t)xb) < nx)
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_walk_events: the reply xids [%d, %d + %llu) cover %d, which ZooKeeper "
                                                   "uses for %s", xb, xb, (unsigned long long)nx, reserved,
                        reserved == -1 ? "watch notifications" : "pings");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    int rc;
    for (Event &e : wk.eev)
        if ((rc = ensure_event(ctx, e)))
            return rc;
    uint32_t launches = 0;
    /* 0. the path table, when the snapshot changed since it was built: timed on its own */
    uint64_t built = 0;
    CK(cudaEventRecord(wk.eev[2], s));
    if ((rc = walk_table(ctx, &built, &launches, who)))
        return rc;
    CK(cudaEventRecord(wk.eev[3], s));
    const uint8_t *ds = bytes;
    if (!in_dev && len) {
        if ((rc = stage_in(ctx, wk.vstream, bytes, len, s)))
            return rc;
        ds = (const uint8_t *)wk.vstream.p;
    }
    const uint64_t nblk = (len + 15) / 16, tiles_s = (nblk + RP_TILE - 1) / RP_TILE;
    const size_t totals_bytes = align16(tiles_s * 4) + (tiles_s / SUPER + 1) * 8;
    if ((rc = ensure_dev(ctx, wk.vword, nblk * 4 + 16)) || (rc = ensure_dev(ctx, wk.vtotals, totals_bytes)) ||
        (rc = ensure_dev(ctx, wk.vtile_base, tiles_s * 8 + 16)) || (rc = ensure_dev(ctx, wk.vcount, EQ_NCOUNTERS * 8)) ||
        (rc = ensure_host(ctx, wk.h_vcount, EQ_NCOUNTERS * 8 + WM_NCOUNTERS * 8)) || (rc = ensure_dev(ctx, wk.zmax, 16)))
        return rc;
    WalkEvParams wp{};
    EvParams &ep = wp.e;
    RepParams &p = ep.r;
    p.s = ds;
    p.len = len;
    p.xid_base = xb;
    p.n = nx;
    p.word = (uint32_t *)wk.vword.p;
    p.tile_total = (uint32_t *)wk.vtotals.p;
    p.super_total = (unsigned long long *)((uint8_t *)wk.vtotals.p + align16(tiles_s * 4));
    p.tile_base = (unsigned long long *)wk.vtile_base.p;
    p.counters = (unsigned long long *)wk.vcount.p;
    ep.start = start;
    unsigned long long *hc = (unsigned long long *)wk.h_vcount.p;
    CK(cudaMemsetAsync(p.counters, 0, EQ_NCOUNTERS * 8, s));
    CK(cudaMemsetAsync(p.tile_total, 0, totals_bytes, s));
    CK(cudaEventRecord(wk.eev[0], s));
    /* 1. the frame chain from `start` (regk_read_events' passes) and where it stops */
    RepParams pf = p;
    const bool sw = wk.gate;                    /* after regk_walk_setwatches: SetWatches replies are frames too */
    if (len > start) {
        if (sw)
            regk_events_sw_cand_kernel<<<(unsigned)tiles_s, RP_TILE, 0, s>>>(ep);
        else
            regk_events_cand_kernel<<<(unsigned)tiles_s, RP_TILE, 0, s>>>(ep);
        CK(cudaGetLastError());
        launches++;
        uint32_t *J = nullptr;
        if ((rc = chain_pass(ctx, &pf, tiles_s, ~0ull, wk.vcand, wk.vmark, wk.vjump, [&](const RepParams &q) {
                regk_children_seed_kernel<<<1, 256, 0, s>>>(q, nullptr, nullptr, 1, start);
            }, &J, &launches, who)))
            return rc;
        if (pf.C) {
            regk_replies_stop_kernel<<<(unsigned)((pf.C + 255) / 256), 256, 0, s>>>(pf);
            CK(cudaGetLastError());
            launches++;
        }
    }
    CK(cudaMemcpyAsync(hc, p.counters, EQ_NCOUNTERS * 8, cudaMemcpyDeviceToHost, s));
    if ((rc = sync_or_fail(ctx, s, who)))
        return rc;
    const uint64_t stop = std::max<uint64_t>(start, hc[RQ_STOP]);
    bool partial = false;
    if (stop < len) {
        /* the first position the chain does not pass: a frame still arriving, or a fault.  Nothing has been marked. */
        uint8_t head[32] = {0};
        const uint64_t avail = len - stop, take = std::min<uint64_t>(avail, sizeof head);
        CK(cudaMemcpyAsync(head, ds + stop, take, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        EvHead h;
        const uint32_t code = sw ? ev_sw_head(head, avail, xb, nx, &h) : ev_head(head, avail, xb, nx, &h);
        if (code != EV_TRUNC)
            return fail(ctx, REGK_ERR_INVALID_ARG, "regk_walk_events: byte %llu: %s (len %d, xid %d)", (unsigned long long)stop,
                code ? events_reason(code) : "internal error", h.len, h.xid);
        partial = true;
    }
    /* 2. the events of the chain mapped against the snapshot as the call found it, then marked */
    const uint64_t C = pf.C;
    if ((rc = ensure_dev(ctx, wk.e_pos, C * 8 + 16)) || (rc = ensure_dev(ctx, wk.e_node, C * 8 + 16)) ||
        (rc = ensure_dev(ctx, wk.e_parent, C * 8 + 16)) || (rc = ensure_dev(ctx, wk.e_zxid, C * 8 + 16)) ||
        (rc = ensure_dev(ctx, wk.e_type, C * 4 + 16)) || (rc = ensure_dev(ctx, wk.e_state, C * 4 + 16)))
        return rc;
    ep.r = pf;
    ep.pos = (unsigned long long *)wk.e_pos.p;
    ep.zxid = (long long *)wk.e_zxid.p;
    ep.type = (int32_t *)wk.e_type.p;
    ep.state = (int32_t *)wk.e_state.p;
    wp.spath = (const uint8_t *)wk.snap_bytes[0].p;
    wp.soff = (const unsigned long long *)wk.snap_off[0].p;
    wp.table = (const uint32_t *)wk.table.p;
    wp.mask = wk.tab_mask;
    wp.mark = (uint32_t *)wk.wmark.p;
    wp.node = (unsigned long long *)wk.e_node.p;
    wp.parent = (unsigned long long *)wk.e_parent.p;
    wp.mcount = (unsigned long long *)wk.mcount.p;
    uint64_t ne = 0;
    if (C) {
        const uint64_t tiles_c = (C + RP_TILE - 1) / RP_TILE;
        const size_t t2 = align16(tiles_c * 4) + (tiles_c / SUPER + 1) * 8;
        if ((rc = ensure_dev(ctx, wk.vntotals, t2)))
            return rc;
        ep.tile_total = (uint32_t *)wk.vntotals.p;
        ep.super_total = (unsigned long long *)((uint8_t *)wk.vntotals.p + align16(tiles_c * 4));
        CK(cudaMemsetAsync(wk.vntotals.p, 0, t2, s));
        regk_events_count_kernel<<<(unsigned)tiles_c, RP_TILE, 0, s>>>(ep);
        regk_walk_events_kernel<<<(unsigned)tiles_c, RP_TILE, 0, s>>>(wp);
        CK(cudaGetLastError());
        launches += 2;
        CK(cudaMemcpyAsync(hc, p.counters, EQ_NCOUNTERS * 8, cudaMemcpyDeviceToHost, s));
        if ((rc = sync_or_fail(ctx, s, who)))
            return rc;
        ne = hc[EQ_NEV];
        if (ne) {
            wp.n_ev = ne;
            regk_walk_mark_kernel<<<(unsigned)((ne + 255) / 256), 256, 0, s>>>(wp);
            CK(cudaGetLastError());
            launches++;
        }
    }
    CK(cudaEventRecord(wk.eev[1], s));
    CK(cudaMemcpyAsync(hc + EQ_NCOUNTERS, wk.mcount.p, WM_NCOUNTERS * 8, cudaMemcpyDeviceToHost, s));
    /* the zxid high-water mark: the chain's replies and SetWatches replies (outside launches and kernel_ms) */
    long long zmax = 0;
    if (C) {
        CK(cudaMemsetAsync(wk.zmax.p, 0, 8, s));
        regk_events_zxid_kernel<<<(unsigned)((C + 255) / 256), 256, 0, s>>>(pf, (long long *)wk.zmax.p);
        CK(cudaGetLastError());
        CK(cudaMemcpyAsync(&zmax, wk.zmax.p, 8, cudaMemcpyDeviceToHost, s));
    }
    if ((rc = sync_or_fail(ctx, s, who)))
        return rc;
    float ms = 0, tms = 0;
    cudaEventElapsedTime(&ms, wk.eev[0], wk.eev[1]);
    cudaEventElapsedTime(&tms, wk.eev[2], wk.eev[3]);
    const void *src[5] = {wk.e_pos.p, wk.e_type.p, wk.e_state.p, wk.e_zxid.p, wk.e_node.p};
    if (!dev_out) {
        HostBuf *hb[5] = {&wk.h_epos, &wk.h_etype, &wk.h_estate, &wk.h_ezxid, &wk.h_enode};
        const size_t sz[5] = {ne * 8, ne * 4, ne * 4, ne * 8, ne * 8};
        for (int k = 0; k < 5; k++) {
            if ((rc = to_host(ctx, *hb[k], src[k], sz[k], s)))
                return rc;
            src[k] = hb[k]->p;
        }
        CK(cudaStreamSynchronize(s));
    }
    wk.n_pending = hc[EQ_NCOUNTERS + WM_PENDING];
    wk.n_removed = hc[EQ_NCOUNTERS + WM_REMOVED];
    wk.zxid = std::max(wk.zxid, zmax);
    out->n_events = ne;
    out->n_pings = hc[EQ_PING];
    out->n_replies = hc[EQ_REPLY];
    out->n_unmatched = hc[EQ_UNMATCHED];
    out->n_other = hc[EQ_OTHER];
    out->consumed = stop;
    out->n_pending = wk.n_pending;
    out->n_removed = wk.n_removed;
    out->table_nodes = built;
    out->partial = partial ? 1u : 0u;
    out->flags = dev_out ? REGK_OUT_DEVICE : 0;
    out->launches = launches;
    out->pos = (const uint64_t *)src[0];
    out->type = (const int32_t *)src[1];
    out->state = (const int32_t *)src[2];
    out->zxid = (const int64_t *)src[3];
    out->node = (const uint64_t *)src[4];
    out->kernel_ms = ms;
    out->table_ms = built ? tms : 0.0f;
    return REGK_OK;
}

int regk_walk_refresh(regk_ctx *ctx, uint32_t flags, regk_walk_refresh_out *out)
{
    const char *who = "regk_walk_refresh";
    if (!ctx || !out)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_walk_refresh: NULL argument");
    memset(out, 0, sizeof *out);
    regk_ctx::Walk &wk = ctx->wk;
    if (flags)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_walk_refresh: flags must be 0");
    if (!wk.active)
        return fail(ctx, REGK_ERR_STATE, "regk_walk_refresh: no walk on this context; call regk_walk_start first");
    if (!wk.watched)
        return fail(ctx, REGK_ERR_STATE, "regk_walk_refresh: the walk is unwatched (a level was framed without "
                                         "REGK_ZK_WATCH); start a new walk with watches");
    if (wk.f)
        return fail(ctx, REGK_ERR_STATE, "regk_walk_refresh: a level is outstanding (the frontier holds %llu nodes); read "
                                         "the walk to its end first", (unsigned long long)wk.f);
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    int rc;
    for (Event &e : wk.ev)
        if ((rc = ensure_event(ctx, e)))
            return rc;
    uint32_t launches = 0;
    const uint64_t m0 = wk.m;
    CK(cudaEventRecord(wk.ev[0], s));
    /* 1. the removed nodes dropped (nothing to do when none is marked) */
    if (wk.n_removed && (rc = walk_rebuild(ctx, nullptr, &launches, who)))
        return rc;
    /* 2. the pending nodes, ascending, as a refresh level's frontier (paths packed from the snapshot); marks cleared */
    const uint64_t m = wk.m, tiles = (m + RP_TILE - 1) / RP_TILE;
    const size_t tb = align16(tiles * 4) + (tiles / SUPER + 1) * 8;
    const int cur = wk.cur;
    if ((rc = ensure_dev(ctx, wk.ktotals, tb)) || (rc = ensure_dev(ctx, wk.kcount, 16)) ||
        (rc = ensure_dev(ctx, wk.xrec, m * 8 + 16)) || (rc = ensure_dev(ctx, wk.fnode, m * 8 + 16)) ||
        (rc = ensure_dev(ctx, wk.flen[cur], m * 4 + 16)))
        return rc;
    uint64_t f = 0, fpt = 0;
    if (m) {
        EvPendParams pp{};
        pp.n = m;
        pp.mark = (const uint32_t *)wk.wmark.p;
        pp.shift = 0;
        pp.epoch = WK_PENDING;
        pp.path_off = (const unsigned long long *)wk.snap_off[0].p;
        pp.tile_total = (uint32_t *)wk.ktotals.p;
        pp.super_total = (unsigned long long *)((uint8_t *)wk.ktotals.p + align16(tiles * 4));
        pp.item = (unsigned long long *)wk.fnode.p;
        pp.rec = (unsigned long long *)wk.xrec.p;
        pp.len = (uint32_t *)wk.flen[cur].p;
        pp.count = (unsigned long long *)wk.kcount.p;
        CK(cudaMemsetAsync(wk.ktotals.p, 0, tb, s));
        regk_events_pending_count_kernel<<<(unsigned)tiles, RP_TILE, 0, s>>>(pp);
        regk_events_pending_kernel<<<(unsigned)tiles, RP_TILE, 0, s>>>(pp);
        CK(cudaGetLastError());
        launches += 2;
        unsigned long long cnt = 0;
        CK(cudaMemcpyAsync(&cnt, pp.count, 8, cudaMemcpyDeviceToHost, s));
        if ((rc = sync_or_fail(ctx, s, who)))
            return rc;
        f = cnt;
        if ((rc = pack_strings(ctx, f, (const uint8_t *)wk.snap_bytes[0].p, pp.path_off, pp.rec, pp.len, wk.gtotals,
                 wk.fbytes[cur], wk.foff[cur], &fpt, &launches)))
            return rc;
        CK(cudaMemsetAsync(wk.wmark.p, 0, m * 4, s));
        CK(cudaMemsetAsync(wk.mcount.p, 0, WM_NCOUNTERS * 8, s));
    }
    CK(cudaEventRecord(wk.ev[1], s));
    if ((rc = sync_or_fail(ctx, s, who)))
        return rc;
    float ms = 0;
    cudaEventElapsedTime(&ms, wk.ev[0], wk.ev[1]);
    wk.n_pending = wk.n_removed = 0;
    wk.f = f;
    wk.fpt = fpt;
    wk.framed = false;
    wk.refreshed = true;
    wk.rlevel = f != 0;
    wk.level_off.assign(1, m);
    out->n_removed = m0 - m;
    out->n_kept = m;
    out->n_frontier = f;
    out->launches = launches;
    out->kernel_ms = ms;
    regk_walk &w = out->walk;
    w.level = 0;
    w.m = m;
    w.n_frontier = f;
    w.level_off = wk.level_off.data();
    w.snapshot.n = m;
    w.snapshot.flags = REGK_IN_DEVICE;
    w.snapshot.path_total = wk.path_total;
    w.snapshot.json_total = wk.data_total;
    w.snapshot.path_bytes = (const uint8_t *)wk.snap_bytes[0].p;
    w.snapshot.path_off = (const uint64_t *)wk.snap_off[0].p;
    w.snapshot.json_bytes = (const uint8_t *)wk.snap_bytes[1].p;
    w.snapshot.json_off = (const uint64_t *)wk.snap_off[1].p;
    w.version = (const int32_t *)wk.ver.p;
    w.ephemeral_owner = (const int64_t *)wk.own.p;
    return REGK_OK;
}

int regk_walk_setwatches(regk_ctx *ctx, const regk_setwatches_opts *o, regk_walk_setwatches_out *out)
{
    const char *who = "regk_walk_setwatches";
    if (!ctx || !o || !out)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_walk_setwatches: NULL argument");
    memset(out, 0, sizeof *out);
    regk_ctx::Walk &wk = ctx->wk;
    if (o->flags & ~(uint32_t)REGK_OUT_DEVICE)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_walk_setwatches: unknown flag bits 0x%x (only REGK_OUT_DEVICE)",
            o->flags & ~(uint32_t)REGK_OUT_DEVICE);
    if (o->max_frame >= 0x80000000u)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_walk_setwatches: max_frame %u is 2^31 or more; a frame's length is a "
                                               "signed 32-bit int", o->max_frame);
    if (!wk.active)
        return fail(ctx, REGK_ERR_STATE, "regk_walk_setwatches: no walk on this context; call regk_walk_start first");
    if (!wk.watched)
        return fail(ctx, REGK_ERR_STATE, "regk_walk_setwatches: the walk is unwatched (a level was framed without "
                                         "REGK_ZK_WATCH); it holds no watches to carry over");
    const uint64_t m = wk.m;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    int rc;
    for (Event &e : wk.swev)
        if ((rc = ensure_event(ctx, e)))
            return rc;
    const unsigned long long *soff = (const unsigned long long *)wk.snap_off[0].p;
    const uint64_t tiles = (m + RP_TILE - 1) / RP_TILE;
    const size_t reg = align16(tiles * 4) + (tiles / SUPER + 1) * 8;
    if ((rc = ensure_dev(ctx, wk.sw_lmax, 16)) || (rc = ensure_dev(ctx, wk.sw_totals, 2 * reg)) ||
        (rc = ensure_dev(ctx, wk.sw_count, 16)) || (rc = ensure_dev(ctx, wk.sw_cls, m + 16)))
        return rc;
    uint32_t launches = 0;
    CK(cudaEventRecord(wk.swev[0], s));
    /* 1. the split's bound: the snapshot's longest path */
    CK(cudaMemsetAsync(wk.sw_lmax.p, 0, 4, s));
    if (m) {
        regk_sw_lmax_kernel<<<(unsigned)((m + 255) / 256), 256, 0, s>>>(soff, m, (uint32_t *)wk.sw_lmax.p);
        CK(cudaGetLastError());
        launches++;
    }
    /* 2. classify: listed or re-pend per node, and the listed nodes' per-tile counts and bytes; nothing is marked yet */
    WalkSwParams wp{};
    wp.m = m;
    wp.path_off = soff;
    wp.armed = (const uint8_t *)wk.armed.p;
    wp.mark = (uint32_t *)wk.wmark.p;
    wp.fnode = (const unsigned long long *)wk.fnode.p;
    wp.f = wk.rlevel ? wk.f : 0;
    wp.cls = (uint8_t *)wk.sw_cls.p;
    for (int k = 0; k < 2; k++) {
        uint8_t *t = (uint8_t *)wk.sw_totals.p + k * reg;
        wp.tt[k] = (uint32_t *)t;
        wp.st[k] = (unsigned long long *)(t + align16(tiles * 4));
    }
    wp.counters = (unsigned long long *)wk.sw_count.p;
    CK(cudaMemsetAsync(wk.sw_totals.p, 0, 2 * reg, s));
    CK(cudaMemsetAsync(wk.sw_count.p, 0, 8, s));
    if (m) {
        regk_walk_sw_classify_kernel<<<(unsigned)tiles, RP_TILE, 0, s>>>(wp);
        CK(cudaGetLastError());
        launches++;
    }
    std::vector<unsigned long long> sup(2 * (tiles / SUPER + 1));
    for (int k = 0; k < 2; k++)
        CK(cudaMemcpyAsync(sup.data() + k * (tiles / SUPER + 1), wp.st[k], (tiles / SUPER + 1) * 8, cudaMemcpyDeviceToHost, s));
    unsigned long long hq[2] = {0, 0};
    uint32_t lmax = 0;
    CK(cudaMemcpyAsync(hq, wk.sw_count.p, 8, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(&lmax, wk.sw_lmax.p, 4, cudaMemcpyDeviceToHost, s));
    if ((rc = sync_or_fail(ctx, s, who)))
        return rc;
    const uint64_t Lmax = 4ull + lmax, mf = o->max_frame ? o->max_frame : 131072u;
    if (mf < SW_OVERHEAD + 2 * Lmax)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_walk_setwatches: max_frame %llu is below this snapshot's minimum of %llu "
                                               "(32 + 2 x (4 + its longest path, %u bytes))", (unsigned long long)mf,
                    (unsigned long long)(SW_OVERHEAD + 2 * Lmax), lmax);
    const uint64_t B = mf - SW_OVERHEAD - Lmax;
    uint64_t nL = 0, bL = 0;
    for (uint64_t q = 0; q <= tiles / SUPER; q++) {
        nL += sup[q];
        bL += sup[tiles / SUPER + 1 + q];
    }
    const uint64_t n_repend = hq[0], ne = 2 * nL, total_s = 2 * bL;
    /* 3. every buffer the rest needs, before any node is re-pended: the last entry starts below total_s, so
       F <= total_s / B + 1 */
    const uint64_t F_max = ne ? total_s / B + 1 : 0, total_max = SW_OVERHEAD * F_max + total_s;
    const bool dev_out = o->flags & REGK_OUT_DEVICE;
    FrameBufs &fb = wk.swframes;
    if ((rc = ensure_dev(ctx, wk.sw_ent_src, ne * 8 + 16)) || (rc = ensure_dev(ctx, wk.sw_ent_s, ne * 8 + 16)) ||
        (rc = ensure_dev(ctx, wk.sw_ent_len, ne * 4 + 16)) || (rc = ensure_dev(ctx, fb.bytes, total_max + 16)) ||
        (rc = ensure_dev(ctx, fb.off, (F_max + 1) * 8)))
        return rc;
    if (!dev_out && ((rc = ensure_host(ctx, fb.h_bytes, total_max + 16)) || (rc = ensure_host(ctx, fb.h_off, (F_max + 1) * 8 + 16))))
        return rc;
    /* 4. place: the entries of D and C, and the re-pend marks */
    wp.nD = nL;
    wp.bD = bL;
    wp.ent_src = (unsigned long long *)wk.sw_ent_src.p;
    wp.ent_s = (unsigned long long *)wk.sw_ent_s.p;
    wp.ent_len = (uint32_t *)wk.sw_ent_len.p;
    if (m) {
        regk_walk_sw_place_kernel<<<(unsigned)tiles, RP_TILE, 0, s>>>(wp);
        CK(cudaGetLastError());
        launches++;
    }
    const unsigned long long mc[WM_NCOUNTERS] = {wk.n_pending + n_repend, wk.n_removed};
    CK(cudaMemcpyAsync(wk.mcount.p, mc, sizeof mc, cudaMemcpyHostToDevice, s));
    uint64_t F = 0;
    if (ne) {
        unsigned long long last_s = 0;
        CK(cudaMemcpyAsync(&last_s, wp.ent_s + (ne - 1), 8, cudaMemcpyDeviceToHost, s));
        if ((rc = sync_or_fail(ctx, s, who)))
            return rc;
        F = last_s / B + 1;
    }
    /* 5. the frames: regk_setwatches_requests' entry writer and frame heads, with E empty */
    const uint64_t total = SW_OVERHEAD * F + total_s;
    SwParams sp{};
    sp.nD = nL;
    sp.nE = 0;
    sp.m = ne;
    sp.bD = bL;
    sp.bE = 0;
    sp.total_s = total_s;
    sp.B = B;
    sp.zxid = wk.zxid;
    sp.ent_src = wp.ent_src;
    sp.ent_s = wp.ent_s;
    sp.ent_len = wp.ent_len;
    sp.path_bytes = (const uint8_t *)wk.snap_bytes[0].p;
    sp.out = (uint8_t *)fb.bytes.p;
    sp.frame_off = (unsigned long long *)fb.off.p;
    sp.F = F;
    if (ne) {
        regk_sw_write_kernel<<<(unsigned)((ne + RP_TILE - 1) / RP_TILE), RP_TILE, 0, s>>>(sp);
        regk_sw_head_kernel<<<(unsigned)((F + 255) / 256), 256, 0, s>>>(sp);
        CK(cudaGetLastError());
        launches += 2;
    } else {
        CK(cudaMemsetAsync(fb.off.p, 0, 8, s));
    }
    CK(cudaEventRecord(wk.swev[1], s));
    const void *src[2] = {fb.bytes.p, fb.off.p};
    if (!dev_out) {
        if ((rc = to_host(ctx, fb.h_bytes, fb.bytes.p, total, s)) || (rc = to_host(ctx, fb.h_off, fb.off.p, (F + 1) * 8, s)))
            return rc;
        src[0] = fb.h_bytes.p;
        src[1] = fb.h_off.p;
    }
    if ((rc = sync_or_fail(ctx, s, who)))
        return rc;
    float ms = 0;
    cudaEventElapsedTime(&ms, wk.swev[0], wk.swev[1]);
    wk.n_pending += n_repend;
    wk.gate = true;
    out->n_listed = nL;
    out->n_repend = n_repend;
    out->n_pending = wk.n_pending;
    out->n_removed = wk.n_removed;
    out->n_frontier = wk.f;
    out->relative_zxid = wk.zxid;
    out->frames.n = F;
    out->frames.total = total;
    out->frames.flags = dev_out ? REGK_OUT_DEVICE : 0;
    out->frames.launches = launches;
    out->frames.frame_bytes = (const uint8_t *)src[0];
    out->frames.frame_off = (const uint64_t *)src[1];
    out->frames.kernel_ms = ms;
    return REGK_OK;
}

int regk_walk_resolve(regk_ctx *ctx, const regk_resolve_opts *o, regk_walk_answers *out)
{
    const char *who = "regk_walk_resolve";
    if (!ctx || !o || !out)
        return fail(ctx, REGK_ERR_INVALID_ARG, "regk_walk_resolve: NULL argument");
    memset(out, 0, sizeof *out);
    ctx->rsv.valid = false;
    regk_ctx::Walk &wk = ctx->wk;
    if (!wk.active)
        return fail(ctx, REGK_ERR_STATE, "%s: no walk on this context; call regk_walk_start first", who);
    regk_decode_in in{};
    in.n = wk.m;
    in.flags = REGK_IN_DEVICE;
    in.path_total = wk.path_total;
    in.json_total = wk.data_total;
    in.path_bytes = (const uint8_t *)wk.snap_bytes[0].p;
    in.path_off = (const uint64_t *)wk.snap_off[0].p;
    in.json_bytes = (const uint8_t *)wk.snap_bytes[1].p;
    in.json_off = (const uint64_t *)wk.snap_off[1].p;
    /* 1. regk_resolve's passes, unchanged: everything but the text */
    ResolveRun r;
    int rc;
    if ((rc = resolve_meta(ctx, &in, o, who, &r)))
        return rc;
    regk_ctx::WalkResolve &wr = ctx->wr;
    cudaStream_t s = ctx->stream;
    const uint64_t m = r.m, T = r.text_total;
    const bool any = o->flags & REGK_RESOLVE_ANY_FORM;
    const bool full = !wr.have || wr.dflt_host != o->default_host_ttl || wr.dflt_srv != o->default_srv_ttl || wr.any != any;
    const int nx = 1 - wr.cur;
    for (Event &ev : wr.ev)
        if ((rc = ensure_event(ctx, ev)))
            return rc;
    if ((rc = ensure_dev(ctx, wr.text[nx], T + 16)) || (rc = ensure_dev(ctx, wr.run[nx], m * 32 + 16)) ||
        (rc = ensure_dev(ctx, wr.text[wr.cur], 16)) || (rc = ensure_dev(ctx, wr.run[wr.cur], 16)))
        return rc;
    /* every host buffer the results need, first: nothing after the stamp can fail on an allocation */
    if (!r.dev_out) {
        regk_ctx::Resolve &rb = ctx->rsv;
        HostBuf *hb[6] = {&rb.h_q_kind, &rb.h_q_node, &rb.h_sec_off, &rb.h_text, &rb.h_cls, &rb.h_unres};
        const size_t sz[6] = {(size_t)r.nq, (size_t)r.nq * 8, (size_t)(2 * r.nq + 1) * 8, (size_t)T, (size_t)m, (size_t)r.n_unres * 8};
        for (int k = 0; k < 6; k++)
            if ((rc = ensure_host(ctx, *hb[k], sz[k] + 16)))
                return rc;
    }
    WalkResolveParams w{};
    w.r = r.p;
    w.r.text = (uint8_t *)wr.text[nx].p;
    w.ident = (const uint32_t *)wk.ident.p;
    w.run_old = (const unsigned long long *)wr.run[wr.cur].p;
    w.run_new = (unsigned long long *)wr.run[nx].p;
    w.ident_out = (uint32_t *)wk.ident.p;
    w.text_total = T;
    uint64_t n_fresh = m, formatted = T, nseg = 0;
    float part = 0;
    const unsigned g2m = (unsigned)((2 * m + 255) / 256);
    if (full) {
        /* 2. nothing to reuse: regk_resolve's emit into this call's text */
        CK(cudaEventRecord(wr.ev[2], s));
        if (m && T) {
            regk_resolve_emit_kernel<<<g2m, 256, 0, s>>>(w.r);
            CK(cudaGetLastError());
            r.launches++;
        }
    } else if (m) {
        /* 2. plan the pieces; 3. segments and scratch offsets */
        const uint64_t n_slots = 4 * m, tiles = (n_slots + RV_TILE - 1) / RV_TILE, nsup = tiles / SUPER + 1;
        const size_t tb = 2 * (tiles + nsup) * 8;
        if ((rc = ensure_dev(ctx, wr.kind, n_slots + 16)) || (rc = ensure_dev(ctx, wr.len, n_slots * 4 + 16)) ||
            (rc = ensure_dev(ctx, wr.src, n_slots * 8 + 16)) || (rc = ensure_dev(ctx, wr.dest, n_slots * 8 + 16)) ||
            (rc = ensure_dev(ctx, wr.totals, tb)) || (rc = ensure_dev(ctx, wr.count, WR_NCOUNTERS * 8)))
            return rc;
        w.n_slots = n_slots;
        w.kind = (uint8_t *)wr.kind.p;
        w.len = (uint32_t *)wr.len.p;
        w.src = (unsigned long long *)wr.src.p;
        w.dest = (unsigned long long *)wr.dest.p;
        unsigned long long *tt = (unsigned long long *)wr.totals.p;
        for (int k = 0; k < 2; k++) {
            w.stile[k] = tt + (size_t)k * (tiles + nsup);
            w.ssuper[k] = w.stile[k] + tiles;
        }
        w.counters = (unsigned long long *)wr.count.p;
        CK(cudaMemsetAsync(wr.kind.p, 0, n_slots, s));
        CK(cudaMemsetAsync(wr.totals.p, 0, tb, s));
        CK(cudaMemsetAsync(wr.count.p, 0, WR_NCOUNTERS * 8, s));
        CK(cudaEventRecord(wr.ev[0], s));
        regk_walk_resolve_plan_kernel<<<g2m, 256, 0, s>>>(w);
        regk_walk_resolve_seg_count_kernel<<<(unsigned)tiles, RV_TILE, 0, s>>>(w);
        CK(cudaGetLastError());
        r.launches += 2;
        CK(cudaEventRecord(wr.ev[1], s));
        std::vector<unsigned long long> sup(2 * nsup + WR_NCOUNTERS);
        for (int k = 0; k < 2; k++)
            CK(cudaMemcpyAsync(sup.data() + k * nsup, w.ssuper[k], nsup * 8, cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(sup.data() + 2 * nsup, w.counters, WR_NCOUNTERS * 8, cudaMemcpyDeviceToHost, s));
        if ((rc = sync_or_fail(ctx, s, who)))
            return rc;
        cudaEventElapsedTime(&part, wr.ev[0], wr.ev[1]);
        r.ms += part;
        formatted = 0;
        for (uint64_t q = 0; q < nsup; q++) {
            nseg += sup[q];
            formatted += sup[nsup + q];
        }
        n_fresh = sup[2 * nsup + WR_C_FRESH_NODES];
        if ((rc = ensure_dev(ctx, wr.seg_src, nseg * 8 + 16)) || (rc = ensure_dev(ctx, wr.seg_dest, nseg * 8 + 16)) ||
            (rc = ensure_dev(ctx, wr.seg_sel, nseg + 16)) || (rc = ensure_dev(ctx, wr.seg_len, nseg * 4 + 16)) ||
            (rc = ensure_dev(ctx, wr.seg_off, (nseg + 1) * 8 + 16)) || (rc = ensure_dev(ctx, wr.scratch, formatted + 16)))
            return rc;
        w.seg_src = (unsigned long long *)wr.seg_src.p;
        w.seg_dest = (unsigned long long *)wr.seg_dest.p;
        w.seg_sel = (uint8_t *)wr.seg_sel.p;
        w.seg_len = (uint32_t *)wr.seg_len.p;
        w.n_seg = nseg;
        w.scratch = (uint8_t *)wr.scratch.p;
        /* 4. the formatted pieces; 5. the text, output-stationary, from the old text and the scratch stream */
        CK(cudaEventRecord(wr.ev[2], s));
        regk_walk_resolve_seg_kernel<<<(unsigned)tiles, RV_TILE, 0, s>>>(w);
        r.launches++;
        if (formatted) {
            regk_walk_resolve_fresh_kernel<<<g2m, 256, 0, s>>>(w);
            r.launches++;
        }
        if (nseg) {
            regk_walk_resolve_seg_len_kernel<<<(unsigned)((nseg + 255) / 256), 256, 0, s>>>(w);
            r.launches++;
        }
        CK(cudaGetLastError());
        uint64_t packed = 0;
        if ((rc = walk_pack(ctx, nseg, (const uint8_t *)wr.text[wr.cur].p, w.scratch, w.seg_src, w.seg_sel, w.seg_len,
                 wr.text[nx], wr.seg_off, &packed, &r.launches)))
            return rc;
        w.r.text = (uint8_t *)wr.text[nx].p;
    } else {
        CK(cudaEventRecord(wr.ev[2], s));
    }
    /* 6. stamp: this call's run offsets and identities, for the next call */
    if (m) {
        regk_walk_resolve_stamp_kernel<<<g2m, 256, 0, s>>>(w);
        CK(cudaGetLastError());
        r.launches++;
    }
    CK(cudaEventRecord(wr.ev[3], s));
    if ((rc = resolve_publish(ctx, r, wr.text[nx].p, wr.ev[2], wr.ev[3], &out->answers, who)))
        return rc;
    ctx->rsv.walk = true;
    ctx->rsv.walk_sgen = wk.sgen;
    wr.cur = nx;
    wr.have = true;
    wr.dflt_host = o->default_host_ttl;
    wr.dflt_srv = o->default_srv_ttl;
    wr.any = any;
    wr.segments = nseg;
    out->n_fresh = n_fresh;
    out->copied_bytes = T - formatted;
    out->formatted_bytes = formatted;
    out->full = full ? 1u : 0u;
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
