"""The stat round against the getData round on 10 M config 3 records (STATS_N overrides), reply streams built on the device,
one registry state for both: every node found, 0.7 % of the payloads rewritten since the baseline (the last byte, so the
length is the same and only mzxid shows it) and 0.3 % of the nodes owned by another session.  In one process the two
rounds alternate five times after a warm-up of each:
  stat     regk_read_stats + regk_reconcile_stats(known_mzxid = the baseline, on the device)
  getdata  regk_read_replies + regk_reconcile_owned
Then the candidate kernel A/B: regk_read_stats with the register form and with the shared-memory form (option
"stats_cand_shared"), alternated five times.  Kernel ms are the library's own events; launches and stream bytes are
counted.  One JSON line per measurement, with the card's name and power limit read in the same run."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from registrar_b200 import _native, synth
from registrar_b200.batch import FLAG_OUT_DEVICE
import replies_util as ru
from test_read_stats import device_stat_replies

N = int(os.environ.get("STATS_N", 10_000_000))
SESSION, OTHER = 0x1234_5678_9ABC_DEF0, 0x0FED_CBA9_8765_4321


def main():
    gpu = torch.cuda.get_device_name(0)
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    card = {"gpu": gpu, "power_limit_max_sm_clock": power}
    ctx = _native.Context(0)
    res = ctx.register_batch(synth.generate("config3", n=N))
    n = res.n
    xs, xg = 1, 1 + n
    ctx.jute_requests(_native.ZK_EXISTS, xid_base=xs, device=True)
    ctx.jute_requests(_native.ZK_GETDATA, xid_base=xg, device=True)
    rng = np.random.default_rng(7)
    perm = rng.permutation(n)
    changed, foreign = perm[:n * 7 // 1000], perm[n * 7 // 1000:n // 100]
    jo = res.json_off.astype(np.int64)
    jb = res.json_bytes.copy()
    jb[jo[changed + 1] - 1] ^= 1
    version = rng.integers(0, 1000, n).astype(np.int32)
    owner = np.full(n, SESSION, np.int64)
    owner[foreign] = OTHER
    known = rng.integers(1, 2 ** 40, n, dtype=np.int64)
    mzxid = known.copy()
    mzxid[changed] += 1
    none = np.zeros(n, bool)
    s_stat, _ = device_stat_replies(n, xs, version, owner, np.diff(jo).astype(np.int32), mzxid, none)
    s_get = ru.device_replies(jb, res.json_off, xg, version, owner, none)
    known_dev = torch.from_numpy(known).cuda()
    del jb, res
    torch.cuda.synchronize()

    def stat_round():
        st = ctx.read_stats(s_stat, device=True)
        d = ctx.reconcile_stats(st, session=SESSION, zk_flags=1, known_mzxid=known_dev, device=True)
        assert (int(d.d.n_update), int(d.n_replace), int(d.d.n_create)) == (changed.size, foreign.size, 0)
        return {"read_ms": float(st.kernel_ms), "reconcile_ms": float(d.d.kernel_ms),
                "launches": int(st.launches) + int(d.d.launches)}

    def getdata_round():
        rep = ctx.read_replies(s_get, device=True)
        cin = rep.snapshot
        stt = _native.CNodeStat(version=rep.version, ephemeral_owner=rep.ephemeral_owner, session=SESSION, zk_flags=1)
        out = _native.CDeltaOwned()
        ctx._check(ctx._lib.regk_reconcile_owned(ctx._h, C.byref(cin), C.byref(stt), FLAG_OUT_DEVICE, C.byref(out)))
        assert (int(out.d.n_update), int(out.n_replace), int(out.d.n_create)) == (changed.size, foreign.size, 0)
        return {"read_ms": float(rep.kernel_ms), "reconcile_ms": float(out.d.kernel_ms),
                "launches": int(rep.launches) + int(out.d.launches)}

    stat_round(), getdata_round()                                       # warm-up: modules loaded, buffers grown
    rows = {"stat": [], "getdata": []}
    for _ in range(5):
        rows["stat"].append(stat_round())
        rows["getdata"].append(getdata_round())
    for name, stream in (("stat", s_stat), ("getdata", s_get)):
        r = rows[name]
        total = [round(x["read_ms"] + x["reconcile_ms"], 3) for x in r]
        print(json.dumps(dict(card, round=name, n=n, stream_bytes=stream.numel(), launches=r[0]["launches"],
                              read_kernel_ms=[round(x["read_ms"], 3) for x in r],
                              reconcile_kernel_ms=[round(x["reconcile_ms"], 3) for x in r], total_kernel_ms=total,
                              best_total_kernel_ms=min(total))), flush=True)
    ab = {0: [], 1: []}
    for shared in (0, 1):
        ctx.set_option("stats_cand_shared", shared)
        ctx.read_stats(s_stat, device=True)
    for _ in range(5):
        for shared in (0, 1):
            ctx.set_option("stats_cand_shared", shared)
            ab[shared].append(round(float(ctx.read_stats(s_stat, device=True).kernel_ms), 3))
    ctx.set_option("stats_cand_shared", 0)
    print(json.dumps(dict(card, ab="read_stats kernel ms by candidate kernel", n=n, stream_bytes=s_stat.numel(),
                          registers=ab[0], shared_memory=ab[1])), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
