/*
 * index.js — drop-in for the registration half of registrar's lib/register.js on top of the N-API addon.
 *
 *   var register = require('registrar-b200').register;     // same (opts, cb) as lib/register.js:174
 *
 * Only the per-record compute changes hands: domainToPath (register.js:34-39), path.join with the hostname
 * (:221-223) and the payload bytes (:141-159) come back from one GPU batch of 1 + aliases records; the
 * ZooKeeper choreography (unlink, 1 s wait, mkdirp, create, put) is the reference's, driven through the same
 * duck-typed opts.zk.  zk.create() receives a Buffer (already-serialised payload) instead of an object.
 *
 * Not runnable in the development image (no Node.js); the Python mirror registrar_b200/registration.py is
 * the tested implementation of exactly this logic.
 */
var os = require('os');
var path = require('path');
var assert = require('assert-plus');
var once = require('once');
var vasync = require('vasync');
var regk = require('./build/Release/regk_napi.node');

var TTL_ABSENT = -2147483648;
var FLAG_NODE_ALIAS = 1 << 2, FLAG_NO_JSON = 1 << 3, FLAG_SKIP_BAD = 1 << 6;

regk.init(0);

function packStrings(strs) {
    var off = Buffer.alloc(4 * (strs.length + 1)), bufs = strs.map(function (s) { return (Buffer.from(s, 'utf8')); });
    var tot = 0;
    bufs.forEach(function (b, i) { tot += b.length; off.writeUInt32LE(tot, 4 * (i + 1)); });
    return ({ bytes: Buffer.concat(bufs), off: off });
}

function toBatch(records, types, flags) {
    var d = packStrings(records.map(function (r) { return (r.domain); }));
    var h = packStrings(records.map(function (r) { return (r.hostname || ''); }));
    var a = packStrings(records.map(function (r) { return (r.address); }));
    var n = records.length;
    var typeId = Buffer.alloc(n), ttl = Buffer.alloc(4 * n), portsOff = Buffer.alloc(4 * (n + 1)),
        present = Buffer.alloc(n), flat = [];
    records.forEach(function (r, i) {
        typeId[i] = types.indexOf(r.type);
        /* out-of-domain numbers are an error, never a silently different payload: the kernels print integers,
           the reference prints any JS number (1.5, 1e21 ...) */
        if (r.ttl !== undefined && (!Number.isInteger(r.ttl) || r.ttl <= TTL_ABSENT || r.ttl > 2147483647))
            throw (new RangeError('record ' + i + ': ttl ' + r.ttl + ' is outside the supported domain (int32)'));
        (r.ports || []).forEach(function (p) {
            if (!Number.isInteger(p) || p < 0 || p > 4294967295)
                throw (new RangeError('record ' + i + ': port ' + p + ' is outside the supported domain (uint32)'));
        });
        ttl.writeInt32LE(r.ttl === undefined ? TTL_ABSENT : r.ttl, 4 * i);
        if (r.ports) { present[i] = 1; flat = flat.concat(r.ports); }
        portsOff.writeUInt32LE(flat.length, 4 * (i + 1));
    });
    var ports = Buffer.alloc(4 * Math.max(flat.length, 1));
    flat.forEach(function (p, i) { ports.writeUInt32LE(p, 4 * i); });
    return ({ n: n, flags: flags, hostStride: 0, domainBytes: d.bytes, domainOff: d.off, hostBytes: h.bytes,
        hostOff: h.off, typeId: typeId, addrBytes: a.bytes, addrOff: a.off, ttl: ttl, portsOff: portsOff,
        ports: ports, portsPresent: present });
}

function slices(bytes, off, n) {
    var out = [], i;
    for (i = 0; i < n; i++)
        out.push(bytes.slice(Number(off.readBigUInt64LE(8 * i)), Number(off.readBigUInt64LE(8 * (i + 1)))));
    return (out);
}

/*
 * registerBatch(records, [opts], cb).  opts.skipBad: a record outside the supported input domain does not fail the
 * batch; out.skipped = [{index, badBits}] lists those records and their paths[i] / payloads[i] are null, for the
 * caller to route to the stock lib/register.js (INTEGRATION.md).
 */
function registerBatch(records, opts, cb) {
    if (typeof (opts) === 'function') { cb = opts; opts = {}; }
    var skip = !!(opts && opts.skipBad);
    var types = [];
    records.forEach(function (r) { if (types.indexOf(r.type) === -1) types.push(r.type); });
    regk.setTypes(types);
    regk.registerBatch(toBatch(records, types, skip ? FLAG_SKIP_BAD : 0), function (err, res) {
        if (err) { cb(err); return; }
        var out = { paths: slices(res.pathBytes, res.pathOff, records.length),
            payloads: slices(res.jsonBytes, res.jsonOff, records.length), kernelMs: res.kernelMs };
        if (skip) {
            out.skipped = [];
            for (var k = 0; k < res.skippedBits.length; k++) {
                var i = Number(res.skippedIndex.readBigUInt64LE(8 * k));
                out.skipped.push({ index: i, badBits: res.skippedBits[k] });
                out.paths[i] = null;
                out.payloads[i] = null;
            }
        }
        cb(null, out);
    });
}

/*
 * N `registration.service` objects -> the payloads of their service records (lib/register.js:45-75), one GPU call.
 * The inner object's key order is kept (JSON.stringify follows insertion order); a missing ttl is 60 and goes last,
 * as the assignment at lib/register.js:197 leaves it.
 */
var SERVICE_KEYS = [ 'srvce', 'proto', 'port', 'ttl' ];

function servicePayloads(services, cb) {
    var n = services.length, port = Buffer.alloc(4 * n), ttl = Buffer.alloc(4 * n), order = Buffer.alloc(n);
    var srv = [], pro = [];
    services.forEach(function (s, i) {
        assert.ok(s.type === 'service');
        var inner = s.service, keys = Object.keys(inner).filter(function (k) { return (k !== 'ttl' || inner.ttl !== undefined); });
        keys.forEach(function (k) {
            if (SERVICE_KEYS.indexOf(k) === -1)
                throw (new RangeError('service ' + i + ': member ' + k + ' is outside the supported domain'));
        });
        if (keys.indexOf('ttl') === -1)
            keys.push('ttl');
        var t = inner.ttl !== undefined ? inner.ttl : 60;
        if (!Number.isInteger(inner.port) || inner.port < 0 || inner.port > 4294967295 || !Number.isInteger(t) ||
            t < -2147483648 || t > 2147483647)
            throw (new RangeError('service ' + i + ': port / ttl outside the supported domain (integers)'));
        srv.push(inner.srvce);
        pro.push(inner.proto);
        port.writeUInt32LE(inner.port, 4 * i);
        ttl.writeInt32LE(t, 4 * i);
        order[i] = keys.reduce(function (acc, k, j) { return (acc | (SERVICE_KEYS.indexOf(k) << (2 * j))); }, 0);
    });
    var s1 = packStrings(srv), p1 = packStrings(pro);
    regk.serviceRecords({ n: n, srvceBytes: s1.bytes, srvceOff: s1.off, protoBytes: p1.bytes, protoOff: p1.off, port: port,
        ttl: ttl, keyOrder: order }, function (err, res) {
        if (err) { cb(err); return; }
        cb(null, slices(res.jsonBytes, res.jsonOff, n));
    });
}

/*
 * The argument contract of register(opts, cb) — reference lib/register.js:175-201 — as data: one row per
 * check, [assert-plus method, path below `options`, only-if path].  Rows run in order, so the first failing
 * check raises the same AssertionError (same method, same label) as the reference does.  Two entries are not
 * plain type checks and are handled by name: 'service.type === service' (register.js:189) and the ttl default
 * (register.js:197), which the reference applies in the middle of the checks.
 */
var CONTRACT = [
    [ 'object', '' ], [ 'object', 'log' ], [ 'optionalString', 'adminIp' ], [ 'optionalObject', 'aliases' ],
    [ 'string', 'domain' ], [ 'object', 'registration' ], [ 'string', 'registration.type' ],
    [ 'optionalNumber', 'registration.ttl' ], [ 'optionalArrayOfNumber', 'registration.ports' ],
    [ 'optionalObject', 'registration.service' ],
    [ 'string', 'registration.service.type', 'registration.service' ],
    [ 'isServiceType', 'registration.service.type', 'registration.service' ],
    [ 'object', 'registration.service.service', 'registration.service' ],
    [ 'string', 'registration.service.service.srvce', 'registration.service' ],
    [ 'string', 'registration.service.service.proto', 'registration.service' ],
    [ 'optionalNumber', 'registration.service.service.ttl', 'registration.service' ],
    [ 'defaultTtl60', 'registration.service.service', 'registration.service' ],
    [ 'number', 'registration.service.service.port', 'registration.service' ],
    [ 'object', 'zk' ]
];

function dig(root, dotted) {
    return (dotted === '' ? root : dotted.split('.').reduce(function (o, k) { return (o[k]); }, root));
}

function checkContract(opts, cb) {
    CONTRACT.forEach(function (row) {
        var how = row[0], where = row[1], onlyIf = row[2];
        if (onlyIf !== undefined && !dig(opts, onlyIf))
            return;
        var v = dig(opts, where), label = where === '' ? 'options' : 'options.' + where;
        if (how === 'isServiceType')
            assert.ok(v === 'service');
        else if (how === 'defaultTtl60')
            v.ttl = v.ttl !== undefined ? v.ttl : 60;
        else
            assert[how](v, label);
    });
    assert.func(cb, 'callback');
}

function register(opts, cb) {
    checkContract(opts, cb);
    cb = once(cb);

    var reg = opts.registration, zk = opts.zk, aliases = opts.aliases || [];
    var ports = reg.ports ? reg.ports : (reg.service ? [ reg.service.service.port ] : undefined);
    var address = opts.adminIp ? opts.adminIp : firstAddress();
    var types = [ reg.type ];
    regk.setTypes(types);
    var host = [ { domain: opts.domain, hostname: os.hostname(), type: reg.type, address: address, ttl: reg.ttl, ports: ports } ];
    var names = [ opts.domain ].concat(aliases).map(function (d) { return ({ domain: d, type: reg.type, address: address }); });
    regk.registerBatch(toBatch(host, types, 0), function (err, h) {
        if (err) { cb(err); return; }
        regk.registerBatch(toBatch(names, types, FLAG_NODE_ALIAS | FLAG_NO_JSON), function (err2, a) {
            if (err2) { cb(err2); return; }
            var aliasPaths = slices(a.pathBytes, a.pathOff, names.length).map(String);
            var cookie = { nodes: [ String(slices(h.pathBytes, h.pathOff, 1)[0]) ].concat(aliasPaths.slice(1)),
                path: aliasPaths[0], payload: slices(h.jsonBytes, h.jsonOff, 1)[0] };
            vasync.pipeline({ arg: cookie, funcs: [
                function cleanup(c, next) {
                    vasync.forEachParallel({ inputs: c.nodes, func: function (n, _cb) {
                        zk.unlink(n, function (e) { _cb(e && e.name !== 'NO_NODE' ? e : undefined); });
                    } }, next);
                },
                function wait(_, next) { setTimeout(once(next), 1000); },
                function mkdirs(c, next) {
                    vasync.forEachParallel({ inputs: c.nodes.map(function (n) { return (path.dirname(n)); }),
                        func: zk.mkdirp.bind(zk) }, next);
                },
                function entries(c, next) {
                    vasync.forEachParallel({ inputs: c.nodes, func: function (n, _cb) {
                        zk.create(n, c.payload, { flags: [ 'ephemeral_plus' ], serialized: true }, once(_cb));
                    } }, next);
                },
                function service(c, next) {
                    if (!reg.service) { next(); return; }
                    /* zk.put(path, obj, cb) has no options argument to flag pre-serialised bytes with, so the
                       object goes to the client as in the reference; servicePayloads() is the batched GPU route
                       (the Python mirror, whose client accepts bytes, uses it inside register()) */
                    zk.put(c.path, { type: 'service', service: reg.service }, function (e) {
                        if (!e && c.nodes.indexOf(c.path) === -1) c.nodes.push(c.path);
                        next(e);
                    });
                }
            ] }, function (e) { if (e) cb(e); else cb(null, cookie.nodes); });
        });
    });
}

function firstAddress() {
    var ifaces = os.networkInterfaces();
    var k = Object.keys(ifaces).filter(function (x) { return (!ifaces[x][0].internal); })[0];
    return (ifaces[k][0].address);
}

module.exports = { register: register, registerBatch: registerBatch, servicePayloads: servicePayloads };
