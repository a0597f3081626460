/*
 * regk.h — C-ABI of libregk.so, the H100-native replacement for registrar's
 * per-record registration hot path (SURVEY.md §8 rows A1–A5).
 *
 * The reference has no FFI of its own (it is 100 % JavaScript); the entry
 * points below are what an N-API addon for that path binds (see
 * INTEGRATION.md and registrar_b200/napi/).  Each one names the reference
 * code it replaces, relative to /root/reference:
 *
 *   regk_register_batch  <- lib/register.js:34-39   domainToPath()            (A1)
 *                           lib/register.js:221-223 path.join(p, hostname)    (A2)
 *                           lib/register.js:141-155 host-record object        (A3)
 *                           lib/register.js:156-159 zk.create(n,_obj,...) ->
 *                             zkplus JSON.stringify(_obj) -> UTF-8 bytes      (A4)
 *                           (new) per-record output offsets                   (A5)
 *   regk_set_types       <- lib/register.js:142,152 `type` / `_obj[type]` key
 *   REGK_NODE_ALIAS      <- lib/register.js:223     aliases.map(domainToPath)
 *
 * Conventions: extern "C", plain pointers and sizes, no exceptions cross the
 * boundary, every call returns a REGK_* status and leaves a message readable
 * through regk_last_error().  There is NO CPU fallback: without a usable
 * CUDA device regk_create() fails.
 *
 * Threading: a context is single-owner (one host thread at a time, one CUDA
 * stream).  The N-API shim runs calls on a napi_async_work thread and
 * resolves the Node errback on the main loop.
 */
#ifndef REGK_H
#define REGK_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define REGK_ABI_VERSION 3

/* ---- status codes ------------------------------------------------------ */
#define REGK_OK                 0
#define REGK_ERR_INVALID_ARG    1   /* NULL pointer, bad flag combination, misaligned device pointer */
#define REGK_ERR_CUDA           2   /* CUDA runtime error; text in regk_last_error() */
#define REGK_ERR_OUT_OF_DOMAIN  3   /* >=1 record outside the fenced input domain; nothing is returned (unless the
                                       batch has REGK_SKIP_BAD: then only REGK_BAD_TOO_LARGE refuses it) */
#define REGK_ERR_NOMEM          4
#define REGK_ERR_STATE          5   /* e.g. type table not set, result already released */

/* ---- batch flags -------------------------------------------------------- */
#define REGK_IN_DEVICE   (1u << 0)  /* batch arrays are device pointers (16-byte aligned); else host memory */
#define REGK_OUT_DEVICE  (1u << 1)  /* result arrays are device pointers; else library-owned pinned host memory */
#define REGK_NODE_ALIAS  (1u << 2)  /* alias nodes: path = domainToPath(domain) un-normalised, no hostname
                                       (lib/register.js:223); default = host nodes (A2, lib/register.js:222) */
#define REGK_NO_JSON     (1u << 3)  /* paths only (skip A3/A4) */
#define REGK_NO_PATH     (1u << 4)  /* payloads only (skip A1/A2) */
#define REGK_JOB_STEP    (1u << 5)  /* this batch is the calling rank's shard of the multi-GPU job bound with
                                       regk_job_bind(): results go straight into every rank's whole-job buffers
                                       (requires REGK_IN_DEVICE | REGK_OUT_DEVICE, paths and payloads) */
#define REGK_SKIP_BAD    (1u << 6)  /* skip mode: a record whose only faults are value-fence bits (REGK_BAD_DOMAIN_BYTE,
                                       _HOST_BYTE, _ADDR_BYTE, _TYPE_ID) gets an empty path and payload (off[i] ==
                                       off[i+1]), every other record is composed exactly as in a batch of the kept records
                                       alone, and the call returns REGK_OK; bad_bits / first_bad then describe the skipped
                                       records and regk_skipped_records() lists them.  REGK_BAD_TOO_LARGE still refuses
                                       the whole batch.  Not with REGK_JOB_STEP.  A clean batch runs exactly the kernels
                                       of a plain one; a dirty one is composed a second time (DESIGN.md section 4) */

/* ---- per-record validation bits (regk_result.bad_bits) ------------------ */
#define REGK_BAD_DOMAIN_BYTE  (1u << 0)  /* byte >= 0x80 or '/' in a domain (JS toLowerCase / path.normalize
                                            semantics are only restated for ASCII, slash-free labels) */
#define REGK_BAD_HOST_BYTE    (1u << 1)  /* hostname empty, ".", "..", or has byte >= 0x80, NUL or '/' */
#define REGK_BAD_ADDR_BYTE    (1u << 2)  /* address empty (a falsy adminIp means auto-detect, register.js:143), or a byte
                                            outside 0x20..0x7f or needing a JSON escape (" or \) */
#define REGK_BAD_TYPE_ID      (1u << 3)  /* type_id >= number of types set */
#define REGK_BAD_TOO_LARGE    (1u << 4)  /* a single record's path or payload exceeds 2^31 bytes */
#define REGK_BAD_SERVICE_BYTE (1u << 5)  /* service records: srvce / proto byte outside 0x20..0x7f or needing a JSON escape */
#define REGK_BAD_KEY_ORDER    (1u << 6)  /* service records: key_order is not a permutation of the four members */

#define REGK_TTL_ABSENT  INT32_MIN      /* registration.ttl === undefined -> key omitted (register.js:144) */

typedef struct regk_ctx regk_ctx;

/*
 * One batch of service records, struct-of-arrays.  All offset arrays are CSR
 * style with n+1 entries, offsets in bytes (or elements for ports_off)
 * relative to the matching *_bytes / ports base.
 */
typedef struct regk_batch {
    uint64_t        n;              /* number of records */
    uint32_t        flags;          /* REGK_IN_DEVICE | REGK_OUT_DEVICE | REGK_NODE_ALIAS | ... */
    uint32_t        host_stride;    /* used when host_off == NULL: hostname i = host_bytes[i*stride, +stride) */

    /* Lengths of the packed arrays (== the last entry of the matching offset array).  Required for
       device-resident batches (the library does not read device memory to size its outputs);
       may be 0 for host batches, the library then reads them from the offset arrays. */
    uint64_t        domain_bytes_len;
    uint64_t        host_bytes_len;
    uint64_t        addr_bytes_len;
    uint64_t        ports_len;      /* elements */

    const uint8_t  *domain_bytes;   /* opts.domain (or one alias) per record, packed */
    const uint32_t *domain_off;     /* [n+1] */

    const uint8_t  *host_bytes;     /* os.hostname() per record (zone UUID in Triton); ignored for alias nodes */
    const uint32_t *host_off;       /* [n+1] or NULL for fixed stride */

    const uint8_t  *type_id;        /* [n] index into the table given to regk_set_types() */

    const uint8_t  *addr_bytes;     /* opts.adminIp per record, packed */
    const uint32_t *addr_off;       /* [n+1] */

    const int32_t  *ttl;            /* [n]; REGK_TTL_ABSENT = undefined */

    const uint32_t *ports_off;      /* [n+1] element offsets into ports, or NULL = no record has ports */
    const uint32_t *ports;          /* registration.ports (or [service.service.port]) values */
    const uint8_t  *ports_present;  /* [n] or NULL.  NULL: ports key present iff k>0.  Non-NULL: !=0 means
                                       present, so an empty array is emitted as "ports":[] (register.js:146) */
} regk_batch;

/*
 * Result views.  path_bytes[path_off[i] .. path_off[i+1]) is znode path i,
 * json_bytes[json_off[i] .. json_off[i+1]) is payload i (what zkplus would
 * hand to ZooKeeper).  Owned by the context until regk_release() or the next
 * regk_register_batch() on the same context with the same result slot.
 */
typedef struct regk_result {
    uint64_t        n;
    uint32_t        flags;          /* REGK_OUT_DEVICE if the pointers below are device pointers */
    uint32_t        bad_bits;       /* OR of REGK_BAD_* over all records (0 on success) */
    uint64_t        first_bad;      /* smallest offending record index when bad_bits != 0 */
    uint8_t        *path_bytes;
    uint64_t       *path_off;       /* [n+1] */
    uint64_t        path_total;     /* == path_off[n] */
    uint8_t        *json_bytes;
    uint64_t       *json_off;       /* [n+1] */
    uint64_t        json_total;     /* == json_off[n] */
    float           kernel_ms;      /* device time of all kernels of the batch (CUDA events on the ctx stream) */
    float           path_kernel_ms; /* regk_path_kernel */
    float           json_kernel_ms; /* regk_json_kernel */
    float           json_len_kernel_ms; /* regk_json_len_kernel (payload lengths + tile bases) */
    uint32_t        launches;       /* kernels launched by this call */
    void           *opaque;         /* library bookkeeping */
    /* REGK_JOB_STEP only: where this rank's shard sits in the job-wide streams and how long those are.  The
       result pointers above are then the rank's own WHOLE-JOB buffers (offsets job-absolute, n_total + 1
       entries); path_total / json_total stay the shard's own byte counts. */
    uint64_t        job_path_base, job_path_total;
    uint64_t        job_json_base, job_json_total;
    uint32_t        generic_tiles;  /* tiles (128 records, counted per kernel) that did not fit the kernels' shared-memory
                                       budget and were composed straight from / to global memory (about 10x slower) */
    uint32_t        reserved;
    /* option "offsets32" = 1 (host results only, both streams below 4 GiB): the offsets come back as 32-bit arrays
       - half the device-to-host bytes of the two offset arrays - and path_off / json_off are NULL */
    uint32_t       *path_off32;     /* [n+1] */
    uint32_t       *json_off32;     /* [n+1] */
} regk_result;

/* ---- lifecycle ----------------------------------------------------------- */
int         regk_abi_version(void);
int         regk_create(int device, regk_ctx **out);   /* binds one CUDA device; fails if none */
void        regk_destroy(regk_ctx *ctx);
const char *regk_last_error(const regk_ctx *ctx);      /* ctx may be NULL: error of the last failed regk_create */

/* Run on a caller-supplied cudaStream_t (e.g. torch's current stream); NULL = the context's own non-blocking
 * stream.  The legacy default stream must be named explicitly (cudaStreamLegacy, (void *)0x1): a NULL here does
 * NOT mean "stream 0", and work on the own stream is not ordered with work on the default stream. */
int         regk_set_stream(regk_ctx *ctx, void *cuda_stream);

/*
 * Record-type table (registration.type values).  Strings are arbitrary UTF-8;
 * JSON escaping (ECMA-262 QuoteJSONString) is applied here, on the host, once.
 * Rejected (REGK_ERR_OUT_OF_DOMAIN): "type", "address", "ttl" (the dynamic key
 * would overwrite a fixed one, register.js:152) and canonical array-index
 * strings ("0", "42": V8 orders integer keys first).
 */
int         regk_set_types(regk_ctx *ctx, const char *const *types, const uint32_t *lens, uint32_t ntypes);

/* ---- the hot path ------------------------------------------------------ */
int         regk_register_batch(regk_ctx *ctx, const regk_batch *batch, regk_result *result);
/* With option "async" = 1 regk_register_batch() only enqueues; regk_finish() waits for that batch,
   fills totals / validation / timings and returns its status.  (Synchronous mode calls it itself.) */
int         regk_finish(regk_ctx *ctx, regk_result *result);
int         regk_release(regk_ctx *ctx, regk_result *result);

/*
 * ---- service records (reference lib/register.js:45-75 registerService) ------------------------------------------
 * The persistent node a registration with `registration.service` also writes: zk.put(domainToPath(domain),
 * { type: 'service', service: registration.service }) with registration.service = { type: 'service', service:
 * { srvce, proto, port, ttl } } (asserted at :186-199, ttl defaulted to 60 at :197).  Payload bytes (zkplus ->
 * JSON.stringify, insertion order):
 *   {"type":"service","service":{"type":"service","service":{<srvce, proto, port, ttl in the CALLER's key order>}}}
 * The node's PATH is an alias-mode path (regk_register_batch with REGK_NODE_ALIAS | REGK_NO_JSON).
 * key_order[i]: four 2-bit key ids, first member in bits 0-1 (0 srvce, 1 proto, 2 port, 3 ttl); NULL = that order.
 * A ttl the caller left undefined is appended last by the reference's assignment: the host layer passes the
 * defaulted value and an order that ends in ttl.  Fence: REGK_BAD_SERVICE_BYTE, REGK_BAD_KEY_ORDER,
 * REGK_BAD_TOO_LARGE (offsets); port is uint32, ttl int32.  Only json_bytes / json_off / json_total of the result
 * are filled.  Synchronous; honours REGK_IN_DEVICE / REGK_OUT_DEVICE.
 */
typedef struct regk_service_batch {
    uint64_t        n;
    uint32_t        flags;
    uint32_t        reserved;
    uint64_t        srvce_bytes_len, proto_bytes_len;   /* required for device batches */
    const uint8_t  *srvce_bytes;    /* registration.service.service.srvce per record, packed ("_http") */
    const uint32_t *srvce_off;      /* [n+1] */
    const uint8_t  *proto_bytes;    /* ....proto ("_tcp") */
    const uint32_t *proto_off;      /* [n+1] */
    const uint32_t *port;           /* [n] */
    const int32_t  *ttl;            /* [n] (already defaulted) */
    const uint8_t  *key_order;      /* [n] or NULL */
} regk_service_batch;

int         regk_service_records(regk_ctx *ctx, const regk_service_batch *batch, regk_result *result);

/*
 * ---- the records a REGK_SKIP_BAD batch skipped ----------------------------------------------------------------
 * Describes the batch finished last on this context, which must have been a skip-mode batch (else REGK_ERR_STATE).
 * The list is compact: a few bad records in 10^7 cost a few bytes, not an n-byte mask.  Downstream calls on "the
 * batch finished last" (regk_parent_dirs, regk_jute_frames / regk_jute_requests, regk_decode with REGK_DECODE_LAST)
 * see the KEPT records in order: their record k is the k-th kept record.  flags: REGK_OUT_DEVICE returns device
 * pointers, otherwise pinned host arrays; both stay valid until the next batch on the context.
 */
typedef struct regk_skipped {
    uint64_t n;                     /* records of the batch */
    uint64_t n_skipped;
    uint32_t flags;                 /* REGK_OUT_DEVICE: device pointers, else pinned host arrays */
    uint32_t bad_bits;              /* OR over the skipped records */
    const uint64_t *index;          /* [n_skipped] ascending record indices */
    const uint8_t  *bits;           /* [n_skipped] REGK_BAD_* of each */
} regk_skipped;

int         regk_skipped_records(regk_ctx *ctx, uint32_t flags, regk_skipped *out);

/* Pinned host memory for callers that want zero-staging H2D/D2H. */
void       *regk_host_alloc(regk_ctx *ctx, size_t bytes);
void        regk_host_free(regk_ctx *ctx, void *p);

/* Device memory helpers for non-CUDA hosts (Node, ctypes). */
void       *regk_dev_alloc(regk_ctx *ctx, size_t bytes);
void        regk_dev_free(regk_ctx *ctx, void *p);
int         regk_memcpy_h2d(regk_ctx *ctx, void *dst_dev, const void *src_host, size_t bytes);
int         regk_memcpy_d2h(regk_ctx *ctx, void *dst_host, const void *src_dev, size_t bytes);
int         regk_sync(regk_ctx *ctx);

/*
 * ---- multi-GPU reassembly (BASELINE.json configs[3]: "sharded across 8 GPUs, all-gather of the output byte
 * stream") ---------------------------------------------------------------------------------------------------
 * One process per GPU; every rank owns whole-job result buffers (regk_dev_alloc) that its peers map through
 * CUDA IPC.  regk_gather_push is an all-gather-v written as ONE kernel over NVLink/NVSwitch peer memory: the
 * calling rank stores its shard's path / payload bytes at their final positions in EVERY rank's buffers
 * (16-byte stores, re-aligned to each destination) and its record offsets rebased by the bytes of the ranks
 * before it.  The reference has no counterpart (one registrar process per host); the operation it replaces is
 * "concatenate the shards' results in record order" (SURVEY.md §8e).
 */
#define REGK_IPC_HANDLE_BYTES 64
#define REGK_MAX_PEERS 16

/* Export a device allocation made by regk_dev_alloc / map a peer's export into this process / unmap it. */
int         regk_ipc_export(regk_ctx *ctx, const void *dev_ptr, unsigned char handle[REGK_IPC_HANDLE_BYTES]);
int         regk_ipc_open(regk_ctx *ctx, const unsigned char handle[REGK_IPC_HANDLE_BYTES], void **peer_ptr);
int         regk_ipc_close(regk_ctx *ctx, void *peer_ptr);

typedef struct regk_gather {
    uint32_t world, rank;
    uint64_t rec_base;              /* records held by the ranks before this one */
    uint64_t n_total;               /* records of the whole job */
    const uint64_t *totals;         /* DEVICE [world][2]: {path bytes, payload bytes} of every rank's shard, as
                                       all-gathered by the caller on the context's stream */
    void *path_bytes[REGK_MAX_PEERS];       /* rank q's whole-job buffers as mapped in THIS process ([rank] = own) */
    uint64_t *path_off[REGK_MAX_PEERS];     /* uint64 [n_total + 1] */
    void *json_bytes[REGK_MAX_PEERS];
    uint64_t *json_off[REGK_MAX_PEERS];
    uint64_t path_cap, json_cap;    /* bytes behind every whole-job byte buffer */
} regk_gather;

/* Enqueue the push of `shard` (a finished REGK_OUT_DEVICE result of this context) on the context's stream.
 * Remote data is complete on a rank once every rank's push has finished: follow it with a stream-ordered
 * barrier across ranks (e.g. a 1-element NCCL all-reduce).  Out-of-range totals raise REGK_ERR_INVALID_ARG
 * at regk_sync time through the returned device flag, never a wild store. */
int         regk_gather_push(regk_ctx *ctx, const regk_result *shard, const regk_gather *g);

/*
 * ---- the multi-GPU job with the all-gather FUSED into the compose kernels ---------------------------------------
 * BASELINE.json configs[3]/[4]: "the record batch shards across the GPUs of one box, one all-gather reassembles
 * the output byte stream".  Here the reassembly is not a separate pass: every rank's regk_path_kernel /
 * regk_json_kernel place each tile at its FINAL position of the job-wide stream and store it, straight out of
 * shared memory (TMA bulk copies, byte-masked at the tile's ragged ends), into the whole-job buffers of ALL ranks
 * over NVLink / NVSwitch, offsets included.  What the ranks must know of each other is two numbers per shard - its
 * path bytes (closed form in the input sizes) and its payload bytes (known after the path kernel's side job) - and
 * those travel through a peer-memory mailbox (regk_peersync.cuh): a 16-byte all-gather + barrier written as a
 * one-warp kernel, no library collective on the data path.  One step on every rank:
 *     exchange(path totals)  ->  regk_path_kernel (push)  ->  exchange(payload totals)  ->  regk_json_kernel (push)
 *     ->  exchange (closing barrier: every rank's stores have landed everywhere)
 * all enqueued on the context's stream by ONE regk_register_batch(REGK_JOB_STEP) call.  The first exchange doubles
 * as the entry barrier: a rank starts overwriting its peers' buffers only after every rank's stream has reached
 * this step, i.e. has finished whatever it had enqueued on the previous step's results.
 * A shard with empty labels (path.join drops them, so the closed-form placement fails) is refused with
 * REGK_ERR_STATE at regk_finish: run it unfused (plain batch + regk_gather_push).
 */
#define REGK_MAILBOX_BYTES (REGK_MAX_PEERS * 32)    /* one 32-byte slot per sender; zero it once after allocation */

typedef struct regk_job {
    uint32_t world, rank;
    uint64_t rec_base;              /* records held by the ranks before this one */
    uint64_t n_total;               /* records of the whole job */
    void *path_bytes[REGK_MAX_PEERS];       /* rank q's whole-job buffers as mapped in THIS process ([rank] = own) */
    uint64_t *path_off[REGK_MAX_PEERS];     /* uint64 [n_total + 1] */
    void *json_bytes[REGK_MAX_PEERS];
    uint64_t *json_off[REGK_MAX_PEERS];
    uint64_t *mailbox[REGK_MAX_PEERS];      /* REGK_MAILBOX_BYTES each, zeroed once */
    uint64_t path_cap, json_cap;    /* bytes behind every whole-job byte buffer */
    uint64_t timeout_ms;            /* how long an exchange waits for a silent peer before failing (0 = 10 s) */
} regk_job;

/* Bind (copy) the job description to the context; NULL unbinds.  No batch may be pending. */
int         regk_job_bind(regk_ctx *ctx, const regk_job *job);

/*
 * ---- setupDirectories for a batch (reference lib/register.js:107-125: mkdirp(path.dirname(n)) for every node) ----
 * Works on the path stream of the batch most recently finished on this context (its device copy is still in
 * the context).  parent_len[i] = byte length of path.dirname(path_i), always a prefix of path_i (node >= 6
 * posix semantics: '/' for a top-level node, '//' when the last separator sits at index 1); unique_first[] =
 * record index of the first occurrence of every DISTINCT directory, ascending - the set a batched mkdirp
 * needs (10^7 instances share ~10^3 parents).  Directories are compared byte for byte; hashing only picks a
 * table slot.  flags: REGK_OUT_DEVICE returns device pointers, otherwise pinned host arrays; both stay valid
 * until the next regk_parent_dirs call on the context.
 */
typedef struct regk_parents {
    uint64_t n;                     /* records of the batch */
    uint64_t n_unique;
    uint32_t flags;
    uint32_t launches;
    const uint32_t *parent_len;     /* [n] */
    const uint64_t *unique_first;   /* [n_unique] */
    float kernel_ms;
} regk_parents;

int         regk_parent_dirs(regk_ctx *ctx, uint32_t flags, regk_parents *out);

/*
 * ---- ZooKeeper wire framing of a batch (reference lib/register.js:156-159: zk.create(n, _obj, {flags:
 * ['ephemeral_plus']}) -> zkplus -> one jute CreateRequest per node on the socket) -----------------------------------
 * Works on the batch most recently finished on this context (paths AND payloads; its device copies are still in
 * the context): frame i = 4-byte big-endian length | RequestHeader{xid = xid_base + i, type = 1 (create)} |
 * CreateRequest{path, data = payload i, acl = [OPEN_ACL_UNSAFE: perms 31, "world", "anyone"], flags = zk_flags}
 * (1 = EPHEMERAL for host records, 0 = persistent for service records).  frame_off[i] = path_off[i] + json_off[i]
 * + 51 i.  PARITY UNPINNED: zkplus / ZooKeeper are not in the reference tree (package.json:20); the layout follows
 * the published zookeeper.jute definitions and is tested against an independent restatement, not against a server.
 * flags: REGK_OUT_DEVICE returns device pointers, else pinned host arrays; valid until the next call.
 */
typedef struct regk_frames {
    uint64_t n;
    uint64_t total;                 /* == frame_off[n] */
    uint32_t flags;
    uint32_t launches;
    const uint8_t *frame_bytes;
    const uint64_t *frame_off;      /* [n+1] */
    float kernel_ms;
} regk_frames;

int         regk_jute_frames(regk_ctx *ctx, uint32_t flags, int32_t xid_base, uint32_t zk_flags, regk_frames *out);

/*
 * The other requests of register()'s choreography, and transactions.  Same batch, same kernel, other framing:
 *   REGK_ZK_CREATE   as regk_jute_frames (lib/register.js:156-159 create; :62 put on a node that does not exist yet)
 *   REGK_ZK_DELETE   DeleteRequest{path, version}: the unlink list of cleanupPreviousEntries (lib/register.js:85-95)
 *                    - one request per node path of the batch, no payload stream needed
 *   REGK_ZK_SETDATA  SetDataRequest{path, data, version}: zkplus put() on an existing node (lib/register.js:62)
 * group = 0: one request per record, xid = xid_base + i.  group = g >= 1: ZooKeeper multi transactions (OpCode 14) of g
 * operations each (the last one may be shorter): frame k = len | xid_base + k | 14 | g x { MultiHeader{op, done = false,
 * err = -1} | request body } | MultiHeader{-1, true, -1} - registering a whole fleet atomically in n / g round trips.
 * out->n = number of frames, frame_off has n + 1 entries.  version is -1 ("any") unless the caller tracks versions.
 * PARITY UNPINNED like regk_jute_frames: restated from zookeeper.jute / MultiTransactionRecord, tested against an
 * independent restatement (oracle/pyoracle.py), not against a server.
 *   REGK_ZK_GETDATA  GetDataRequest{path, watch = false}: the heartbeat's read of every node (lib/zk.js:21-44), whose
 *                    replies regk_read_replies turns into a snapshot.  Frame i = len | xid_base + i (wrapping) | 4 | path
 *                    length | path | 0, 17 + P_i bytes.  Paths only; group != 0 is REGK_ERR_INVALID_ARG (a multi holds
 *                    no reads).  A successful call records the batch, xid_base and n for regk_read_replies.
 */
#define REGK_ZK_CREATE  1u
#define REGK_ZK_DELETE  2u
#define REGK_ZK_GETDATA 4u
#define REGK_ZK_SETDATA 5u

typedef struct regk_jute_opts {
    uint32_t op;                    /* REGK_ZK_* */
    uint32_t flags;                 /* REGK_OUT_DEVICE */
    int32_t xid_base;
    uint32_t zk_flags;              /* create: CreateMode bits (1 = EPHEMERAL) */
    int32_t version;                /* delete / setData: expected version, -1 = any */
    uint32_t group;                 /* 0: single requests; g >= 1: multi transactions of g operations */
} regk_jute_opts;

int         regk_jute_requests(regk_ctx *ctx, const regk_jute_opts *opts, regk_frames *out);

/*
 * ---- the whole mkdirp set of a batch (reference lib/register.js:107-129: zk.mkdirp(path.dirname(n)) for every node;
 * mkdirp creates the directory AND every ancestor, and ZooKeeper creates no node whose parent is missing) -----------
 * Works on the path stream of the batch finished last, as regk_parent_dirs does: a skip-mode batch contributes its
 * kept records in order; a REGK_NO_PATH batch, an empty batch (it leaves no path stream), a REGK_JOB_STEP result or a
 * pending batch is REGK_ERR_STATE.
 * D_i = path.dirname(path_i) (parent_len of regk_parent_dirs).  D_i == "/" creates nothing.  D_i is INVALID when
 * ZooKeeper's path check rejects it - an empty component ("//"), a trailing '/', or a byte in 0x00-0x1F or 0x7F
 * (only alias nodes with empty labels and domains with control bytes get there): it contributes nothing and its
 * first record is listed in invalid[].  Every other D_i contributes each of its prefixes that ends at a component
 * boundary: /a, /a/b, ..., D_i.  The set is the union, each directory once, in a deterministic order: ascending
 * depth (components), then ascending first record whose directory has it as a prefix - every parent precedes its
 * children, so the whole list can be pipelined on one session.  Directory k = path_{dir_rec[k]}[0, dir_len[k]), also
 * packed as dir_bytes[dir_off[k], dir_off[k+1]).  Bytes are compared byte for byte; a hash only picks a table slot.
 * flags: REGK_OUT_DEVICE returns device pointers, else pinned host arrays; they stay valid until the next
 * regk_mkdirp_dirs call (a later batch does not touch them).  Option "mkdirp_tight_table" = 1 shrinks the hash table
 * to the smallest power of two above the entry count (long probe chains; for testing).
 */
typedef struct regk_dirs {
    uint64_t n;                     /* records of the batch */
    uint64_t n_dirs;                /* directories to create */
    uint64_t n_invalid;             /* distinct immediate directories ZooKeeper would reject */
    uint32_t flags;                 /* REGK_OUT_DEVICE */
    uint32_t launches;
    uint32_t max_depth;
    uint32_t reserved;
    const uint64_t *dir_rec;        /* [n_dirs] first record whose directory has this one as a prefix */
    const uint32_t *dir_len;        /* [n_dirs] */
    const uint64_t *depth_off;      /* [max_depth + 1] depth d is directories depth_off[d-1] .. depth_off[d]; [0] = 0 */
    const uint8_t  *dir_bytes;      /* [dir_bytes_len] packed directory paths */
    const uint64_t *dir_off;        /* [n_dirs + 1] */
    const uint64_t *invalid;        /* [n_invalid] first record of each rejected directory, ascending */
    uint64_t dir_bytes_len;
    float kernel_ms;                /* parent_ms + closure_ms + gather_ms */
    float parent_ms;                /* the distinct immediate directories (regk_parents.cuh kernels) */
    float closure_ms;               /* classify + every depth's passes, including the host's read of two counters per depth */
    float gather_ms;                /* dir_off and dir_bytes */
} regk_dirs;

int         regk_mkdirp_dirs(regk_ctx *ctx, uint32_t flags, regk_dirs *out);

/*
 * The mkdirp set of the last regk_mkdirp_dirs call (REGK_ERR_STATE without one) as ready-to-send frames: directory k
 * becomes len | RequestHeader{xid = xid_base + k (wrapping), type = 1} | CreateRequest{path, data = empty buffer
 * (length 0), acl = [OPEN_ACL_UNSAFE], flags = zk_flags}, in set order - the same kernel and layout as
 * regk_jute_requests(REGK_ZK_CREATE, group = 0).  Single requests only: a multi transaction would abort as a whole on
 * the first directory that already exists, and a NODE_EXISTS reply to one of these frames is expected (zkplus'
 * mkdirp tolerates it).  PARITY UNPINNED: the data bytes and flags zkplus' own mkdirp sends are not in the reference
 * tree (zkplus is a dependency, package.json:20), hence an empty buffer and zk_flags as a parameter (0 = persistent).
 * flags: REGK_OUT_DEVICE returns device pointers, else pinned host arrays; valid until the next call.  These buffers
 * are separate from regk_jute_requests', so the create frames of the batch and the mkdirp frames can be held together.
 */
int         regk_mkdirp_requests(regk_ctx *ctx, int32_t xid_base, uint32_t zk_flags, uint32_t flags, regk_frames *out);

/*
 * ---- the reader side: decode paths and payloads back into records (README.md:462-480, :587-664) -----------------
 * Inverse of regk_register_batch / regk_service_records for audits of registry contents and round-trip checks:
 *   path    -> domain (labels reversed back, '/' -> '.'); for host nodes the last component is the instance name
 *              (lib/register.js:221-223) and is reported as (host_pos, host_len) inside the path
 *   payload -> type, address (positions inside the payload), ttl, ports - for the canonical compact form
 *              {"type":T,"address":A[,"ttl":n],T:{"address":A[,"ports":[..]]}} ; service records
 *              {"type":"service","service":{"type":"service","service":{srvce,proto,port,ttl in any order}}} come
 *              back with type_* = srvce, addr_* = proto, ports[0] = port.
 * Input: explicit streams (host, or device with REGK_IN_DEVICE; 64-bit CSR offsets as in regk_result), or
 * REGK_DECODE_LAST = the batch finished last on this context.  Either stream may be NULL.
 * Output: rec[n]; domains in SLOT layout (domain i = dom_bytes[path_off[i], + rec[i].dom_len)); ports in slot layout
 * (record i's ports = ports[json_off[i] / 2, + rec[i].nports)).  REGK_OUT_DEVICE returns device pointers.
 */
#define REGK_DECODE_LAST       (1u << 8)

#define REGK_DEC_PATH_OK        (1u << 0)
#define REGK_DEC_HOST_RECORD    (1u << 1)
#define REGK_DEC_SERVICE_RECORD (1u << 2)
#define REGK_DEC_NOT_CANONICAL  (1u << 3)   /* not the compact form this library writes */
#define REGK_DEC_KEY_MISMATCH   (1u << 4)   /* the inner object's name differs from the value of "type" (README.md:596) */
#define REGK_DEC_ADDR_MISMATCH  (1u << 5)   /* the two "address" members differ */
#define REGK_DEC_BAD_NUMBER     (1u << 6)   /* ttl / port not an integer in range */
#define REGK_DEC_BAD_PATH       (1u << 7)   /* no leading '/', or a host node without an instance name */

typedef struct regk_decoded {
    uint32_t flags;                 /* REGK_DEC_* */
    uint32_t dom_len;
    uint32_t host_pos, host_len;    /* instance name inside the path (host nodes) */
    uint32_t type_pos, type_len;    /* inside the payload (JSON escapes left as they are) */
    uint32_t addr_pos, addr_len;
    int32_t  ttl;                   /* REGK_TTL_ABSENT when the key is missing */
    uint32_t nports;                /* 0xFFFFFFFF when the key is missing */
} regk_decoded;

typedef struct regk_decode_in {
    uint64_t n;
    uint32_t flags;                 /* REGK_IN_DEVICE | REGK_OUT_DEVICE | REGK_DECODE_LAST */
    uint32_t host_nodes;            /* != 0: paths are host nodes (domain path + '/' + instance name) */
    uint64_t path_total, json_total;    /* required for device streams */
    const uint8_t *path_bytes;
    const uint64_t *path_off;       /* [n+1] */
    const uint8_t *json_bytes;
    const uint64_t *json_off;       /* [n+1] */
} regk_decode_in;

typedef struct regk_decode_out {
    uint64_t n;
    uint32_t flags;
    uint32_t launches;
    const regk_decoded *rec;        /* [n] */
    const uint8_t *dom_bytes;       /* [path_total] slot layout */
    const uint32_t *ports;          /* [json_total / 2 + 1] slot layout */
    uint64_t dom_bytes_len, ports_len;
    float kernel_ms;
} regk_decode_out;

int         regk_decode(regk_ctx *ctx, const regk_decode_in *in, regk_decode_out *out);

/*
 * ---- reconcile a batch with a snapshot of the registry (the batch form of the reference's heartbeat check,
 * lib/zk.js:21-44 and lib/index.js:55-159: stat every node, register again what is missing) ----------------------
 * Desired = the batch finished last on this context, as for regk_jute_requests: paths AND payloads required; a
 * skip-mode batch contributes its kept records in order; no batch, a REGK_NO_PATH / REGK_NO_JSON batch, an empty batch
 * (it leaves no streams), a REGK_JOB_STEP result or a pending batch is REGK_ERR_STATE.
 * Observed = a snapshot of m nodes (path j, data j) in the layout regk_decode accepts: host streams, or device streams
 * with REGK_IN_DEVICE (bytes 4-byte aligned, offsets 8-byte aligned); u64 CSR offsets; path_total / json_total are
 * required for device streams; host_nodes is ignored, REGK_DECODE_LAST is REGK_ERR_INVALID_ARG.  Offsets that are not
 * monotone or reach past the totals are REGK_ERR_INVALID_ARG naming the smallest bad node (host snapshots are checked
 * on the host, device snapshots by the first kernel before any byte of that node is read).  A snapshot in which two
 * nodes have the same path is malformed (a registry cannot hold that): REGK_ERR_INVALID_ARG naming the later node.
 * The snapshot must cover exactly the namespace the batch owns: every node it holds that the batch does not produce -
 * directories included - is classed DELETE.
 * Nodes are keyed by their path bytes, compared byte for byte (a hash only picks a table slot); the class depends on
 * bytes alone (no ephemeral owners, no versions) - regk_reconcile_owned below also weighs each node's Stat.  Record i:
 *   REGK_DELTA_DUP     an earlier record of the batch has the same path (the first occurrence decides); no request
 *   REGK_DELTA_CREATE  no node has path i
 *   REGK_DELTA_UPDATE  the node with path i holds data that differs from payload i in length or in a byte
 *   REGK_DELTA_SAME    the node with path i holds payload i
 * match[i] = that node's index or UINT64_MAX (DUP records carry their path's match too).  Node j: REGK_DELTA_KEEP if
 * some record has path j, else REGK_DELTA_DELETE.  create / update / dup list record indices, del snapshot indices,
 * all ascending.  n and m must be < 2^32 - 1.  flags: REGK_OUT_DEVICE returns device pointers, else pinned host
 * arrays; valid until the next regk_reconcile call.
 * The call also gathers the three request sets (create paths + payloads, update paths + payloads, delete paths) into
 * streams of the library's own, so regk_reconcile_requests needs neither the snapshot nor the batch afterwards; a later
 * batch does not touch them.  Option "reconcile_tight_table" = 1 sizes both hash tables to the smallest power of two
 * above their entry count (long probe chains; for testing).
 */
#define REGK_DELTA_SAME   0u        /* cls[] */
#define REGK_DELTA_CREATE 1u
#define REGK_DELTA_UPDATE 2u
#define REGK_DELTA_DUP    3u
#define REGK_DELTA_KEEP   0u        /* obs_cls[] */
#define REGK_DELTA_DELETE 1u

typedef struct regk_delta {
    uint64_t n, m;                  /* records of the batch finished last / nodes of the snapshot */
    uint64_t n_same, n_create, n_update, n_dup, n_delete;
    uint32_t flags, launches;       /* REGK_OUT_DEVICE */
    const uint8_t  *cls;            /* [n] REGK_DELTA_SAME / _CREATE / _UPDATE / _DUP */
    const uint64_t *match;          /* [n] */
    const uint8_t  *obs_cls;        /* [m] REGK_DELTA_KEEP / _DELETE */
    const uint64_t *create, *update, *dup;   /* ascending record indices */
    const uint64_t *del;            /* [n_delete] ascending snapshot indices */
    float kernel_ms;
} regk_delta;

int         regk_reconcile(regk_ctx *ctx, const regk_decode_in *snapshot, uint32_t flags, regk_delta *out);

/*
 * The requests that repair the registry, from the last regk_reconcile call (REGK_ERR_STATE without one), framed
 * exactly as regk_jute_requests frames a batch: frame k is list entry k (group = 0) or multi transaction k, xid =
 * xid_base + k; group, version and zk_flags mean what they mean there.
 *   REGK_ZK_CREATE   the create list: CreateRequest{path i, payload i}
 *   REGK_ZK_SETDATA  the update list: SetDataRequest{path i, payload i, version}
 *   REGK_ZK_DELETE   the delete list: DeleteRequest{snapshot path j, version}
 * Send them in this order: delete, then the creates' parents (regk_mkdirp_dirs / regk_mkdirp_requests), then create,
 * then setData, then (after regk_reconcile_owned) replace.  flags: REGK_OUT_DEVICE returns device pointers, else pinned
 * host arrays; valid until the next call.  The frames come from whichever of regk_reconcile / regk_reconcile_owned last
 * succeeded.  After regk_reconcile_owned two more options exist:
 *   REGK_ZK_REPLACE           (op) the replace list: frame q is one multi transaction (group = 0 counts as 1; at most
 *                             32768 entries, i.e. 65536 operations) - len | xid_base + q | 14 | for each entry (record i):
 *                             MultiHeader{2, false, -1} DeleteRequest{path i, version} MultiHeader{1, false, -1}
 *                             CreateRequest{path i, payload i, [OPEN_ACL_UNSAFE], zk_flags} | MultiHeader{-1, true, -1}.
 *                             Entry r is 65 + 2 P + J bytes, a frame 21 more.  The node is never missing: ZooKeeper applies
 *                             the delete and the create together or neither.
 *   REGK_ZK_VERSION_OBSERVED  (flags) every delete, setData and the delete of a replace carries the Stat.version its
 *                             node had in the snapshot instead of opts->version: the write fails with BADVERSION if the
 *                             node changed since.  Not with REGK_ZK_CREATE (REGK_ERR_INVALID_ARG).
 * Both are REGK_ERR_STATE after a plain regk_reconcile.  After regk_reconcile_owned, REGK_ZK_CREATE and REGK_ZK_REPLACE
 * require opts->zk_flags == the zk_flags the reconcile classified with (REGK_ERR_INVALID_ARG otherwise): a node created
 * in another mode would be classed REPLACE again by the next reconcile, and the repair would never converge.
 */
#define REGK_ZK_REPLACE          256u       /* regk_jute_opts.op: not a ZooKeeper OpCode */
#define REGK_ZK_VERSION_OBSERVED (1u << 9)  /* regk_jute_opts.flags */

int         regk_reconcile_requests(regk_ctx *ctx, const regk_jute_opts *opts, regk_frames *out);

/*
 * ---- reconcile against node stats: ephemeral owners and versions (the reference re-registers after a session loss by
 * unlinking every node, waiting 1 s and creating it again, lib/register.js:85-95, :228-239) ----------------------------
 * As regk_reconcile, with the Stat of every snapshot node, as the caller's client read it (getData / exists replies):
 * version[j] = Stat.version, ephemeral_owner[j] = Stat.ephemeralOwner (0 = persistent).  The arrays live where the
 * snapshot's streams do (device arrays with REGK_IN_DEVICE: version 4-byte, ephemeral_owner 8-byte aligned).
 * want = session when zk_flags == 1 (EPHEMERAL), else 0.  Record i is REGK_DELTA_REPLACE when it is the first record
 * with its path, node j has that path and ephemeral_owner[j] != want - a stale ephemeral of an earlier session (which
 * the server would delete when that session expires), another session's ephemeral, or a persistent node where an
 * ephemeral is wanted (and the reverse).  The payload is not compared then.  Every other class is as in regk_reconcile;
 * the node of a REPLACE record is KEEP (its delete travels inside the replace frame).
 * n_same + n_create + n_update + n_dup + n_replace == n.
 * Edge: a persistent node that has children, where an ephemeral is wanted, is REPLACE too; ZooKeeper then aborts the
 * multi with NOTEMPTY, as the reference's unlink fails there.  An ephemeral node has no children, so the reverse cannot.
 * Refused besides regk_reconcile's refusals (REGK_ERR_INVALID_ARG): stat NULL, an array NULL while m > 0, misaligned
 * device arrays, zk_flags other than 0 or 1 (a sequential or container mode makes a path key meaningless), zk_flags == 1
 * with session == 0.  The delta's arrays are valid until the next regk_reconcile / regk_reconcile_owned call.
 */
typedef struct regk_node_stat {
    const int32_t *version;         /* [m] Stat.version of snapshot node j (passed through verbatim) */
    const int64_t *ephemeral_owner; /* [m] Stat.ephemeralOwner of node j; 0 = persistent */
    int64_t  session;               /* session id the repair will be sent on */
    uint32_t zk_flags;              /* CreateMode of the batch's nodes: 1 = EPHEMERAL, 0 = persistent; nothing else */
    uint32_t reserved;
} regk_node_stat;

#define REGK_DELTA_REPLACE 4u       /* cls[]: only regk_reconcile_owned produces it */

typedef struct regk_delta_owned {
    regk_delta d;                   /* filled as regk_reconcile fills it; cls[] may hold REGK_DELTA_REPLACE */
    uint64_t n_replace;
    const uint64_t *replace;        /* [n_replace] ascending record indices */
} regk_delta_owned;

int         regk_reconcile_owned(regk_ctx *ctx, const regk_decode_in *snapshot, const regk_node_stat *stat,
                                 uint32_t flags, regk_delta_owned *out);

/*
 * ---- the replies to the getData frames of a batch, as a snapshot (the input half of the heartbeat: lib/zk.js:21-44
 * stats every node, lib/index.js:131-159; and of re-registration after a session loss, lib/register.js:85-95,
 * :228-239) -------------------------------------------------------------------------------------------------------------
 * bytes[0, len) = what the caller read off the session after sending the frames of the last REGK_ZK_GETDATA
 * regk_jute_requests call, back to back, from the first reply's length word on; host memory, or device memory with
 * REGK_IN_DEVICE in flags (16-byte aligned).  Frame = int len | ReplyHeader{int xid; long zxid; int err} | body, big
 * endian; body = GetDataResponse{buffer data (D = -1: null, read as empty); Stat (68 bytes)} when err == 0 (len == 88 +
 * max(D, 0)), none otherwise (len == 16).  ZooKeeper answers a session's requests in order: the k-th frame that is not
 * a watch notification (xid -1) or a ping (xid -2) must carry xid == xid_base + k (wrapping) and answers record k.
 * Notifications and pings met before the n-th reply are skipped and counted; the stream may go on past the n-th reply.
 * n_found + n_missing + n_error == n.  err[k] = ReplyHeader.err of record k's reply.
 * snapshot: one node per distinct path among the replies with err == 0 (the first such reply gives it; later ones with
 * the same path are dropped, as regk_reconcile refuses a snapshot that repeats a path; paths are compared byte for byte,
 * a hash only picks a table slot).  Node j = record node_rec[j]: its path from the batch, its data from the reply, its
 * Stat.version and Stat.ephemeralOwner - exactly the input regk_reconcile_owned(ctx, &out->snapshot, {version,
 * ephemeral_owner, session, zk_flags}, ...) takes.  The snapshot holds the batch's own paths only, so a reconcile against
 * it lists no DELETE.  A record whose reply is NONODE (-101) gets no node, so reconcile classes it CREATE; so does a
 * record whose reply carries any other error: do not send the repair while n_error > 0.
 * err and node_rec are pinned host arrays, or device arrays with REGK_OUT_DEVICE; the snapshot, version and
 * ephemeral_owner are always device arrays.  All stay valid until the next regk_read_replies call (a later batch does
 * not touch them).
 * REGK_ERR_STATE: no REGK_ZK_GETDATA framing since the batch finished last, a batch finished since that framing, or a
 * pending batch.  REGK_ERR_INVALID_ARG (the message names the byte position and the expected xid): the stream ends
 * before the n-th reply is complete (and says how many were), len < 16, a negative xid other than -1 / -2, an xid
 * outside the framed range, a reply out of order or for a record that already has one, a success frame whose length
 * disagrees with its data length, D < -1, Stat.dataLength != max(D, 0), an error reply with a body; an xid range
 * [xid_base, xid_base + n) that covers -1 or -2; NULL pointers; a misaligned device stream.
 * PARITY UNPINNED: the reply layout is restated from zookeeper.jute and tested against an independent restatement.
 */
typedef struct regk_replies {
    uint64_t n;                     /* requests: records of the framed batch */
    uint64_t m;                     /* snapshot nodes: one per distinct path among replies with err == 0 */
    uint64_t n_found, n_missing, n_error;   /* replies with err 0 / NONODE (-101) / any other err */
    uint64_t n_skipped;             /* watch notifications (xid -1) and pings (xid -2) met before the n-th reply */
    uint64_t consumed;              /* stream bytes up to the end of the n-th reply */
    uint32_t flags, launches;
    const int32_t  *err;            /* [n] ReplyHeader.err of record i's reply; REGK_OUT_DEVICE decides host/device */
    const uint64_t *node_rec;       /* [m] record whose reply gave node j, ascending; same side as err */
    regk_decode_in  snapshot;       /* ALWAYS device (REGK_IN_DEVICE set): path j = that record's path from the batch,
                                       data j = the reply's data; aligned as regk_reconcile requires */
    const int32_t  *version;        /* [m] device: Stat.version */
    const int64_t  *ephemeral_owner;/* [m] device: Stat.ephemeralOwner */
    float kernel_ms;
} regk_replies;

int         regk_read_replies(regk_ctx *ctx, const uint8_t *bytes, uint64_t len, uint32_t flags, regk_replies *out);

/* Tuning knobs (kernel variant selection for A/B measurement); see DESIGN.md. */
int         regk_set_option(regk_ctx *ctx, const char *name, int64_t value);
int64_t     regk_get_option(const regk_ctx *ctx, const char *name);

#ifdef __cplusplus
}
#endif
#endif /* REGK_H */
