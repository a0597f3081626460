"""regk_read_children on two workloads, with the getChildren reply stream built on the device from the batch:
  fleet   tests/test_mkdirp_set.py's fleet (4 M config 2 records under 1 000 domains), every directory listing its
          instances plus 1 % extra stale children (a copy of an instance name with '~' appended);
  config3 10 M config 3 records, about one child per directory, every child an instance of the batch.
Each is read from a device stream five times (best kernel_ms).  Prints one JSON line per workload with kernel ms,
launches, stream bytes, children and stale counts, and the card's name and power limit read in the same run."""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from registrar_b200 import _native, synth


def fleet(n, ndom=1000, seed=3):
    """n config 2 records collapsed onto the domains of the first `ndom` (tests/test_mkdirp_set.py)"""
    rng = np.random.default_rng(seed)
    b = synth.generate("config2", n=n)
    idx = rng.integers(0, ndom, n)
    lens = np.diff(b.domain_off)[idx]
    off = np.zeros(n + 1, np.uint32)
    np.cumsum(lens, out=off[1:])
    src0 = b.domain_off[:-1][idx]
    pos = np.repeat(src0.astype(np.int64) - off[:-1].astype(np.int64), lens) + np.arange(int(off[-1]), dtype=np.int64)
    b.domain_bytes = b.domain_bytes[pos]
    b.domain_off = off
    return b


def children_stream(res, parent_len, xid_base, stale_frac, seed=1):
    """GetChildrenResponse frames, one per distinct directory in order of first record, listing every record's name
    (and, for a fraction of records, a stale copy), built on the device.  Returns (CUDA uint8 tensor, d, entries)."""
    n = res.n
    po = res.path_off.astype(np.int64)
    pb = res.path_bytes.tobytes()
    ids, dir_of = {}, np.empty(n, np.int64)
    for i in range(n):
        key = pb[po[i]:po[i] + int(parent_len[i])]
        dir_of[i] = ids.setdefault(key, len(ids))
    d = len(ids)
    rng = np.random.default_rng(seed)
    extra = np.flatnonzero(rng.random(n) < stale_frac)
    rec = np.concatenate([np.arange(n), extra])                         # entry -> record
    tilde = np.concatenate([np.zeros(n, bool), np.ones(len(extra), bool)])
    order = np.argsort(dir_of[rec], kind="stable")
    rec, tilde = rec[order], tilde[order]
    edir = dir_of[rec]
    name_off = po[rec] + parent_len[rec].astype(np.int64) + 1
    L = po[rec + 1] - name_off + tilde
    cnt = np.bincount(edir, minlength=d)
    body = np.zeros(d, np.int64)
    np.add.at(body, edir, 4 + L)
    flen = 24 + body
    foff = np.zeros(d + 1, np.int64)
    np.cumsum(flen, out=foff[1:])
    # entry positions: frame start + 24 + the sizes of the entries before it in its frame
    esz = 4 + L
    ecum = np.cumsum(esz) - esz
    first = np.zeros(d, np.int64)
    first[1:] = np.cumsum(cnt)[:-1]
    epos = foff[edir] + 24 + ecum - ecum[first[edir]]
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    out = torch.zeros(int(foff[-1]), dtype=torch.uint8, device="cuda")
    be = lambda v: torch.from_numpy(np.ascontiguousarray(np.asarray(v, np.int64).astype(">i4")).view(np.uint8).reshape(-1, 4))
    head = torch.zeros((d, 24), dtype=torch.uint8)
    head[:, 0:4] = be(flen - 4)
    head[:, 4:8] = be((xid_base + np.arange(d) + 2 ** 31) % 2 ** 32 - 2 ** 31)
    head[:, 20:24] = be(cnt)
    out[(dev(foff[:-1])[:, None] + torch.arange(24, device="cuda")[None, :]).reshape(-1)] = head.cuda().reshape(-1)
    out[(dev(epos)[:, None] + torch.arange(4, device="cuda")[None, :]).reshape(-1)] = be(L).cuda().reshape(-1)
    src = dev(np.frombuffer(pb, np.uint8))
    Lc, no, ep = dev(L - tilde), dev(name_off), dev(epos + 4)
    rep = torch.repeat_interleave(torch.arange(len(rec), device="cuda"), Lc)
    start = torch.cumsum(Lc, 0) - Lc
    within = torch.arange(rep.numel(), device="cuda") - start[rep]
    out[ep[rep] + within] = src[no[rep] + within]
    t = torch.from_numpy(np.flatnonzero(tilde)).cuda()
    out[ep[t] + Lc[t]] = ord("~")
    return out, d, len(rec)


def measure(ctx, name, batch, stale_frac):
    res = ctx.register_batch(batch)
    parent_len, _, _ = ctx.parent_dirs()
    ctx.children_requests(_native.ZK_GETCHILDREN, xid_base=1, device=True)
    stream, d, entries = children_stream(res, parent_len, 1, stale_frac)
    del res
    torch.cuda.synchronize()
    runs = []
    for _ in range(5):
        t0 = time.perf_counter()
        r = ctx.read_children(stream, device=True)
        runs.append(((time.perf_counter() - t0) * 1e3, float(r.kernel_ms)))
    assert int(r.n_dirs) == d and int(r.n_children) == entries and int(r.consumed) == stream.numel()
    return {"workload": name, "n": batch.n, "dirs": d, "children": entries, "stale": int(r.n_stale),
            "stream_bytes": stream.numel(), "launches": int(r.launches),
            "kernel_ms": [round(k, 3) for _, k in runs], "wall_ms": [round(w, 3) for w, _ in runs],
            "best_kernel_ms": round(min(k for _, k in runs), 3)}


def main():
    scale = float(sys.argv[1]) if len(sys.argv) > 1 else 1.0
    gpu = torch.cuda.get_device_name(0)
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    ctx = _native.Context(0)
    for name, batch, frac in (("fleet", fleet(int(4_000_000 * scale)), 0.01),
                              ("config3", synth.generate("config3", n=int(10_000_000 * scale)), 0.0)):
        row = measure(ctx, name, batch, frac)
        row.update(gpu=gpu, power_limit_max_sm_clock=power)
        print(json.dumps(row), flush=True)
        torch.cuda.empty_cache()
    ctx.close()


if __name__ == "__main__":
    main()
