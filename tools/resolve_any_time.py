"""REGK_RESOLVE_ANY_FORM's cost on tools/resolve_time.py's fleet (4 M config 2 records under 1 000 service records), as
device snapshots in three forms:
  canonical  as the library composes them, resolved without and with the flag (the candidate passes on a clean registry)
  pretty     every node pretty-printed in the README's layout (two-space indent, one member per line), with the flag
  general1   1 % of the nodes pretty-printed, with the flag
Runs are alternated in one process, five rounds; best kernel_ms per variant.  The reader's share comes from a
torch.profiler pass of its own (regk_resolve_any_read_kernel's device time over the whole call's).  Prints one JSON line
per variant and the card's name and power limit read in the same run."""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from registrar_b200 import _native
from registrar_b200.batch import Snapshot
from resolve_time import SERVICE, fleet


def readme_layout(d: bytes) -> bytes:
    """a compact record laid out as the README prints its records: one member per line, two-space indent per level"""
    out, depth, in_str, k = bytearray(), 0, False, 0
    while k < len(d):
        c = d[k]
        if in_str:
            out.append(c)
            if c == 0x5C:
                out.append(d[k + 1])
                k += 1
            elif c == 0x22:
                in_str = False
        elif c == 0x22:
            in_str = True
            out.append(c)
        elif c in b"{[":
            depth += 1
            out += bytes([c]) + b"\n" + b"  " * depth
        elif c in b"}]":
            depth -= 1
            out += b"\n" + b"  " * depth + bytes([c])
        elif c == 0x2C:
            out += b",\n" + b"  " * depth
        elif c == 0x3A:
            out += b": "
        else:
            out.append(c)
        k += 1
    return bytes(out) + b"\n"


def snapshots(res, idx):
    """(canonical, pretty, general1) device snapshots of the batch's nodes and one service record per domain"""
    po, jo = res.path_off.astype(np.int64), res.json_off.astype(np.int64)
    _, first = np.unique(idx, return_index=True)
    dirs = []
    for i in first.tolist():
        p = res.path_bytes[po[i]:po[i + 1]].tobytes()
        dirs.append(p[:p.rfind(b"/")])
    pb = np.concatenate([res.path_bytes[:int(po[-1])], np.frombuffer(b"".join(dirs), np.uint8)])
    po2 = np.concatenate([po, po[-1] + np.cumsum([len(d) for d in dirs])])
    jbs = res.json_bytes[:int(jo[-1])].tobytes()
    payloads = [jbs[jo[j]:jo[j + 1]] for j in range(len(jo) - 1)] + [SERVICE] * len(dirs)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    out = []
    for every in (0, 1, 100):
        ps = payloads if not every else [readme_layout(d) if j % every == 0 else d for j, d in enumerate(payloads)]
        jb = np.frombuffer(b"".join(ps), np.uint8)
        jo2 = np.zeros(len(ps) + 1, np.int64)
        np.cumsum([len(d) for d in ps], out=jo2[1:])
        out.append(Snapshot(t(pb), t(po2), t(jb), t(jo2)))
    return out


def reader_share(ctx, snap):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ctx.resolve(snap, 30, 60, device=True, any_form=True)
        torch.cuda.synchronize()
    tot, rd = 0.0, 0.0
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
        if "regk_" in e.key:
            tot += us
            if "any_read" in e.key:
                rd += us
    return round(rd / 1e3, 3), round(tot / 1e3, 3)


def main():
    scale = float(sys.argv[1]) if len(sys.argv) > 1 else 1.0
    gpu = torch.cuda.get_device_name(0)
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    ctx = _native.Context(0)
    b, idx = fleet(int(4_000_000 * scale))
    res = ctx.register_batch(b)
    canon, pretty, general1 = snapshots(res, idx)
    del res
    variants = [("canonical", canon, False), ("canonical+flag", canon, True), ("pretty+flag", pretty, True),
                ("general1%+flag", general1, True)]
    check = {}
    for name, snap, flag in variants:                       # warm-up, and every variant's answers
        a = ctx.resolve(snap, 30, 60, any_form=flag)
        check[name] = (a.text.tobytes(), a.node_cls.tobytes(), int(a.launches))
    same = all(check[n][:2] == check["canonical"][:2] for n, _, _ in variants)
    times = {n: [] for n, _, _ in variants}
    for _ in range(5):
        for name, snap, flag in variants:
            times[name].append(float(ctx.resolve(snap, 30, 60, device=True, any_form=flag).kernel_ms))
    for name, snap, flag in variants:
        row = {"variant": name, "m": snap.m, "json_bytes": snap.json_bytes.numel(), "launches": check[name][2],
               "kernel_ms": [round(x, 3) for x in times[name]], "best_kernel_ms": round(min(times[name]), 3),
               "answers_equal_canonical": same, "gpu": gpu, "power_limit_max_sm_clock": power}
        if flag:
            row["reader_ms"], row["profiled_total_ms"] = reader_share(ctx, snap)
        print(json.dumps(row), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
