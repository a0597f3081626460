/*
 * regk_napi.c — thin N-API addon over the C-ABI (include/regk.h): what BASELINE.json's north_star calls
 * "a thin N-API C-ABI addon".  It only marshals: every record byte is produced by libregk.so's kernels.
 *
 *   const regk = require('./build/Release/regk_napi.node');
 *   regk.setTypes(['host', 'load_balancer', ...]);
 *   regk.registerBatch({n, flags, hostStride, domainBytes, domainOff, hostBytes, hostOff?, typeId,
 *                       addrBytes, addrOff, ttl, portsOff?, ports?, portsPresent?},  // Buffers over SoA arrays
 *                      function (err, res) { res.pathBytes, res.pathOff, res.jsonBytes, res.jsonOff, res.kernelMs });
 *   flags may include REGK_SKIP_BAD (1 << 6): out-of-domain records come back empty and res.skippedIndex (u64 LE) /
 *   res.skippedBits (u8) list them (regk_skipped_records).
 *   regk.serviceRecords({n, srvceBytes, srvceOff, protoBytes, protoOff, port, ttl, keyOrder?},
 *                       function (err, res) { res.jsonBytes, res.jsonOff });          // regk_service_records
 *
 * Threading (SURVEY.md §8b): the context is single-owner, but libuv runs queued napi_async_work items on a POOL
 * of worker threads, so two registerBatch() calls can execute at the same time.  Everything that touches the
 * context therefore happens inside job_execute under one mutex: the job's own copy of the type table is
 * installed if it differs from the one the context holds, the batch runs, and the results are copied out of
 * the library's recycled pinned buffers into memory the job owns — all before the lock is released.  The main
 * thread never calls into the context (setTypes only records the table for the jobs queued after it); the
 * errback fires on the main loop, like every callback in the reference.
 *
 * Build (on a machine with Node.js; not possible in the image this repo is developed in — no node, no
 * node_api.h): node-gyp with `libraries: ['-lregk']`, or
 *   gcc -shared -fPIC -I$(node -p "process.execPath+'/../../include/node'") -I../../include \
 *       -o regk_napi.node regk_napi.c -L.. -lregk
 */
#ifdef REGK_NAPI_MIN_DECLS
#include "napi_min.h"
#else
#include <node_api.h>
#endif
#include <pthread.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/regk.h"

static regk_ctx *g_ctx;
static pthread_mutex_t g_lock = PTHREAD_MUTEX_INITIALIZER;     /* serialises every use of g_ctx (worker threads) */

/* an immutable, reference-counted type table: setTypes() publishes one, every job pins the one current when
   it is queued (main thread only touches g_types / refcounts under g_lock as well) */
typedef struct {
    int refs;
    uint32_t n;
    char **strs;
    uint32_t *lens;
} types_t;
static types_t *g_types;            /* what setTypes() recorded last */
static types_t *g_installed;        /* what the context holds (compared by identity) */

static void types_unref(types_t *t)
{
    uint32_t i;
    int dead;
    if (!t)
        return;
    pthread_mutex_lock(&g_lock);
    dead = --t->refs == 0;
    pthread_mutex_unlock(&g_lock);
    if (!dead)
        return;
    for (i = 0; i < t->n; i++)
        free(t->strs[i]);
    free(t->strs);
    free(t->lens);
    free(t);
}

static const void *buf_or_null(napi_env env, napi_value obj, const char *name, size_t *len)
{
    napi_value v;
    void *data = NULL;
    size_t n = 0;
    if (napi_get_named_property(env, obj, name, &v) != napi_ok || napi_get_buffer_info(env, v, &data, &n) != napi_ok)
        data = NULL, n = 0;
    if (len)
        *len = n;
    return data;
}

static uint32_t u32_prop(napi_env env, napi_value obj, const char *name)
{
    napi_value v;
    uint32_t x = 0;
    if (napi_get_named_property(env, obj, name, &v) == napi_ok)
        napi_get_value_uint32(env, v, &x);
    return x;
}

typedef struct {
    regk_batch batch;
    regk_service_batch svc;             /* serviceRecords(): this one is used instead of `batch` */
    int is_service;
    regk_result result;
    int status;
    char error[512];
    napi_ref cb, keepalive;             /* the batch object: keeps the Buffers alive while the worker runs */
    napi_async_work work;
    types_t *types;                     /* pinned at queue time */
    /* the job's own copies of the results (made under the lock, handed to V8 as external buffers) */
    uint8_t *path_bytes, *json_bytes;
    uint64_t *path_off, *json_off;
    uint64_t n_skipped;                 /* REGK_SKIP_BAD: the skipped records, copied like the results */
    uint64_t *skip_index;
    uint8_t *skip_bits;
} job_t;

static void *dup_bytes(const void *p, size_t n)
{
    void *q = malloc(n ? n : 1);
    if (q && n)
        memcpy(q, p, n);
    return q;
}

static void free_hint(napi_env env, void *data, void *hint)
{
    (void)env;
    (void)hint;
    free(data);
}

static void job_execute(napi_env env, void *data)
{
    job_t *j = (job_t *)data;
    (void)env;
    pthread_mutex_lock(&g_lock);
    j->status = REGK_OK;
    if (j->types && j->types != g_installed) {
        j->status = regk_set_types(g_ctx, (const char *const *)j->types->strs, j->types->lens, j->types->n);
        if (j->status == REGK_OK)
            g_installed = j->types;     /* identity only; the job's own reference keeps it alive while it matters */
    }
    if (j->status == REGK_OK)
        j->status = j->is_service ? regk_service_records(g_ctx, &j->svc, &j->result)
                                  : regk_register_batch(g_ctx, &j->batch, &j->result);  /* host buffers in, pinned host buffers out */
    if (j->status != REGK_OK) {
        strncpy(j->error, regk_last_error(g_ctx), sizeof j->error - 1);
    } else {
        const size_t noff = (size_t)(j->result.n + 1) * 8;
        j->path_bytes = (uint8_t *)dup_bytes(j->result.path_bytes, (size_t)j->result.path_total);
        j->json_bytes = (uint8_t *)dup_bytes(j->result.json_bytes, (size_t)j->result.json_total);
        j->path_off = j->result.path_off ? (uint64_t *)dup_bytes(j->result.path_off, noff) : (uint64_t *)calloc(1, noff);
        j->json_off = (uint64_t *)dup_bytes(j->result.json_off, noff);
        regk_release(g_ctx, &j->result);
        if (!j->is_service && (j->batch.flags & REGK_SKIP_BAD)) {
            regk_skipped sk;
            j->status = regk_skipped_records(g_ctx, 0, &sk);
            if (j->status == REGK_OK) {
                j->n_skipped = sk.n_skipped;
                j->skip_index = (uint64_t *)dup_bytes(sk.index, (size_t)sk.n_skipped * 8);
                j->skip_bits = (uint8_t *)dup_bytes(sk.bits, (size_t)sk.n_skipped);
            } else {
                strncpy(j->error, regk_last_error(g_ctx), sizeof j->error - 1);
            }
        }
        if (j->status == REGK_OK && (!j->path_bytes || !j->json_bytes || !j->path_off || !j->json_off ||
                ((j->batch.flags & REGK_SKIP_BAD) && !j->is_service && (!j->skip_index || !j->skip_bits)))) {
            j->status = REGK_ERR_NOMEM;
            strncpy(j->error, "out of memory copying the results", sizeof j->error - 1);
        }
    }
    if (g_installed == j->types && j->status != REGK_OK && j->types)
        g_installed = NULL;             /* be conservative after a failure: the next job re-installs its table */
    pthread_mutex_unlock(&g_lock);
}

static void job_complete(napi_env env, napi_status st, void *data)
{
    job_t *j = (job_t *)data;
    napi_value cb, undef, argv[2], res, v;
    (void)st;
    napi_get_reference_value(env, j->cb, &cb);
    napi_get_undefined(env, &undef);
    if (j->status != REGK_OK) {
        napi_value msg;
        napi_create_string_utf8(env, j->error, strlen(j->error), &msg);
        napi_create_error(env, NULL, msg, &argv[0]);
        if (j->status == REGK_ERR_OUT_OF_DOMAIN) {
            napi_create_double(env, (double)j->result.first_bad, &v);
            napi_set_named_property(env, argv[0], "firstBad", v);
            napi_create_double(env, (double)j->result.bad_bits, &v);
            napi_set_named_property(env, argv[0], "badBits", v);
        }
        napi_call_function(env, undef, cb, 1, argv, NULL);
    } else {
        const uint64_t n = j->result.n;
        napi_get_null(env, &argv[0]);
        napi_create_object(env, &res);
        /* the job's own copies (made under the lock in job_execute); V8 frees them with the Buffers */
        napi_create_external_buffer(env, (size_t)j->result.path_total, j->path_bytes, free_hint, NULL, &v);
        napi_set_named_property(env, res, "pathBytes", v);
        napi_create_external_buffer(env, (size_t)(n + 1) * 8, j->path_off, free_hint, NULL, &v);
        napi_set_named_property(env, res, "pathOff", v);
        napi_create_external_buffer(env, (size_t)j->result.json_total, j->json_bytes, free_hint, NULL, &v);
        napi_set_named_property(env, res, "jsonBytes", v);
        napi_create_external_buffer(env, (size_t)(n + 1) * 8, j->json_off, free_hint, NULL, &v);
        napi_set_named_property(env, res, "jsonOff", v);
        j->path_bytes = j->json_bytes = NULL;
        j->path_off = j->json_off = NULL;
        napi_create_double(env, (double)j->result.kernel_ms, &v);
        napi_set_named_property(env, res, "kernelMs", v);
        if (j->skip_index) {
            napi_create_external_buffer(env, (size_t)j->n_skipped * 8, j->skip_index, free_hint, NULL, &v);
            napi_set_named_property(env, res, "skippedIndex", v);
            napi_create_external_buffer(env, (size_t)j->n_skipped, j->skip_bits, free_hint, NULL, &v);
            napi_set_named_property(env, res, "skippedBits", v);
            j->skip_index = NULL;
            j->skip_bits = NULL;
        }
        argv[1] = res;
        napi_call_function(env, undef, cb, 2, argv, NULL);
    }
    free(j->path_bytes);
    free(j->json_bytes);
    free(j->path_off);
    free(j->json_off);
    free(j->skip_index);
    free(j->skip_bits);
    types_unref(j->types);
    napi_delete_reference(env, j->cb);
    napi_delete_reference(env, j->keepalive);
    napi_delete_async_work(env, j->work);
    free(j);
}

static napi_value register_batch(napi_env env, napi_callback_info info)
{
    size_t argc = 2, len;
    napi_value argv[2], name;
    job_t *j;
    napi_get_cb_info(env, info, &argc, argv, NULL, NULL);
    if (argc < 2 || !g_ctx) {
        napi_throw_error(env, NULL, "registerBatch(batch, cb): init() first, two arguments required");
        return NULL;
    }
    j = (job_t *)calloc(1, sizeof *j);
    j->batch.n = u32_prop(env, argv[0], "n");
    j->batch.flags = u32_prop(env, argv[0], "flags") & ~(REGK_IN_DEVICE | REGK_OUT_DEVICE);
    j->batch.host_stride = u32_prop(env, argv[0], "hostStride");
    j->batch.domain_bytes = (const uint8_t *)buf_or_null(env, argv[0], "domainBytes", &len);
    j->batch.domain_off = (const uint32_t *)buf_or_null(env, argv[0], "domainOff", NULL);
    j->batch.host_bytes = (const uint8_t *)buf_or_null(env, argv[0], "hostBytes", NULL);
    j->batch.host_off = (const uint32_t *)buf_or_null(env, argv[0], "hostOff", NULL);
    j->batch.type_id = (const uint8_t *)buf_or_null(env, argv[0], "typeId", NULL);
    j->batch.addr_bytes = (const uint8_t *)buf_or_null(env, argv[0], "addrBytes", NULL);
    j->batch.addr_off = (const uint32_t *)buf_or_null(env, argv[0], "addrOff", NULL);
    j->batch.ttl = (const int32_t *)buf_or_null(env, argv[0], "ttl", NULL);
    j->batch.ports_off = (const uint32_t *)buf_or_null(env, argv[0], "portsOff", NULL);
    j->batch.ports = (const uint32_t *)buf_or_null(env, argv[0], "ports", NULL);
    j->batch.ports_present = (const uint8_t *)buf_or_null(env, argv[0], "portsPresent", NULL);
    pthread_mutex_lock(&g_lock);
    j->types = g_types;
    if (j->types)
        j->types->refs++;
    pthread_mutex_unlock(&g_lock);
    napi_create_reference(env, argv[0], 1, &j->keepalive);
    napi_create_reference(env, argv[1], 1, &j->cb);
    napi_create_string_utf8(env, "regk_register_batch", 19, &name);
    napi_create_async_work(env, NULL, name, job_execute, job_complete, j, &j->work);
    napi_queue_async_work(env, j->work);
    return NULL;
}

/* serviceRecords({n, srvceBytes, srvceOff, protoBytes, protoOff, port, ttl, keyOrder?}, cb): payloads of the
   persistent service nodes (lib/register.js:45-75) - res.jsonBytes / res.jsonOff; the paths come from registerBatch
   with the alias flag */
static napi_value service_records(napi_env env, napi_callback_info info)
{
    size_t argc = 2;
    napi_value argv[2], name;
    job_t *j;
    napi_get_cb_info(env, info, &argc, argv, NULL, NULL);
    if (argc < 2 || !g_ctx) {
        napi_throw_error(env, NULL, "serviceRecords(batch, cb): init() first, two arguments required");
        return NULL;
    }
    j = (job_t *)calloc(1, sizeof *j);
    j->is_service = 1;
    j->svc.n = u32_prop(env, argv[0], "n");
    j->svc.srvce_bytes = (const uint8_t *)buf_or_null(env, argv[0], "srvceBytes", NULL);
    j->svc.srvce_off = (const uint32_t *)buf_or_null(env, argv[0], "srvceOff", NULL);
    j->svc.proto_bytes = (const uint8_t *)buf_or_null(env, argv[0], "protoBytes", NULL);
    j->svc.proto_off = (const uint32_t *)buf_or_null(env, argv[0], "protoOff", NULL);
    j->svc.port = (const uint32_t *)buf_or_null(env, argv[0], "port", NULL);
    j->svc.ttl = (const int32_t *)buf_or_null(env, argv[0], "ttl", NULL);
    j->svc.key_order = (const uint8_t *)buf_or_null(env, argv[0], "keyOrder", NULL);
    napi_create_reference(env, argv[0], 1, &j->keepalive);
    napi_create_reference(env, argv[1], 1, &j->cb);
    napi_create_string_utf8(env, "regk_service_records", 20, &name);
    napi_create_async_work(env, NULL, name, job_execute, job_complete, j, &j->work);
    napi_queue_async_work(env, j->work);
    return NULL;
}

static napi_value set_types(napi_env env, napi_callback_info info)
{
    /* Main thread: only RECORDS the table.  It reaches the context inside the next job's job_execute, under
       the lock, so a batch already running on a worker keeps the table it was queued with. */
    size_t argc = 1;
    napi_value argv[1], el;
    uint32_t n = 0, i;
    types_t *t, *old;
    napi_get_cb_info(env, info, &argc, argv, NULL, NULL);
    if (argc < 1 || napi_get_array_length(env, argv[0], &n) != napi_ok) {
        napi_throw_error(env, NULL, "setTypes(types): an array of strings is required");
        return NULL;
    }
    t = (types_t *)calloc(1, sizeof *t);
    t->refs = 1;
    t->n = n;
    t->strs = (char **)calloc(n ? n : 1, sizeof *t->strs);
    t->lens = (uint32_t *)calloc(n ? n : 1, sizeof *t->lens);
    for (i = 0; i < n; i++) {
        size_t l = 0;
        napi_get_element(env, argv[0], i, &el);
        napi_get_value_string_utf8(env, el, NULL, 0, &l);
        t->strs[i] = (char *)malloc(l + 1);
        napi_get_value_string_utf8(env, el, t->strs[i], l + 1, &l);
        t->lens[i] = (uint32_t)l;
    }
    pthread_mutex_lock(&g_lock);
    old = g_types;
    g_types = t;
    pthread_mutex_unlock(&g_lock);
    types_unref(old);
    return NULL;
}

static napi_value init_ctx(napi_env env, napi_callback_info info)
{
    size_t argc = 1;
    napi_value argv[1];
    uint32_t device = 0;
    napi_get_cb_info(env, info, &argc, argv, NULL, NULL);
    if (argc >= 1)
        napi_get_value_uint32(env, argv[0], &device);
    if (!g_ctx && regk_create((int)device, &g_ctx) != REGK_OK)
        napi_throw_error(env, NULL, regk_last_error(NULL));     /* no CUDA device: no CPU fallback */
    return NULL;
}

static napi_value module_init(napi_env env, napi_value exports)
{
    napi_property_descriptor props[] = {
        { "init", NULL, init_ctx, NULL, NULL, NULL, 0, NULL },
        { "setTypes", NULL, set_types, NULL, NULL, NULL, 0, NULL },
        { "registerBatch", NULL, register_batch, NULL, NULL, NULL, 0, NULL },
        { "serviceRecords", NULL, service_records, NULL, NULL, NULL, 0, NULL },
    };
    napi_define_properties(env, exports, sizeof props / sizeof props[0], props);
    return exports;
}

NAPI_MODULE(regk_napi, module_init)
