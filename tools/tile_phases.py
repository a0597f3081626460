"""Where a compose CTA's time goes: per-CTA phase stamps of regk_path_kernel and regk_json_kernel.

Builds libregk.so with the product's nvcc flags plus -DREGK_PHASE_STAMPS (into a temporary directory, or takes a
library built that way with --lib), loads it through REGK_LIB and runs device-resident batches as bench.py does:
two batches of --records records, rotated.  Thread 0 of every CTA stamps clock64() at

  path kernel     0 start, 1 plan barrier passed, 2 bytes landed, 3 composed (after the tail barrier), 4 end
  payload kernel  0 start, 1 metadata and length in registers, 2 scan done (and fragment table landed),
                  3 composed (after the tail barrier), 4 end

("end" is after cp.async.bulk.wait_group.read).  Prints median and p90 of every phase in microseconds at the SM
clock NVML reports during the run, the card and its power limit, and how many CTAs of each kernel an SM held at
once (from the stamps: the most at any moment, and the average over the kernel's span on that SM).  One JSON line.
"""
import argparse
import json
import os
import sys
import tempfile
import threading

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PHASES = {
    "path": [("plan", 0, 1), ("landed", 1, 2), ("prologue", 0, 2), ("compose", 2, 3), ("flush", 3, 4), ("life", 0, 4)],
    "json": [("meta", 0, 1), ("scan", 1, 2), ("prologue", 0, 2), ("compose", 2, 3), ("flush", 3, 4), ("life", 0, 4)],
}


def build_instrumented(out_dir):
    import subprocess
    import __graft_entry__ as g
    so = os.path.join(out_dir, "libregk_phases.so")
    subprocess.check_call([g.NVCC] + g.NVCC_FLAGS + ["-DREGK_PHASE_STAMPS", "-o", so,
                                                     os.path.join(g.CSRC, "regk_api.cu")])
    return so


class Clock(threading.Thread):
    """SM clock (MHz) sampled through NVML every 5 ms while `active` is set."""

    def __init__(self):
        super().__init__(daemon=True)
        import pynvml
        pynvml.nvmlInit()
        self.nv = pynvml
        vis = os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]
        self.h = pynvml.nvmlDeviceGetHandleByIndex(int(vis) if vis.isdigit() else 0)
        self.samples, self.active, self.stop = [], threading.Event(), threading.Event()

    def run(self):
        while not self.stop.is_set():
            if self.active.wait(0.05):
                self.samples.append(self.nv.nvmlDeviceGetClockInfo(self.h, self.nv.NVML_CLOCK_SM))
                self.stop.wait(0.005)

    def card(self):
        name = self.nv.nvmlDeviceGetName(self.h)
        return {"name": name.decode() if isinstance(name, bytes) else name,
                "power_limit_w": self.nv.nvmlDeviceGetPowerManagementLimit(self.h) / 1000.0,
                "sm_max_mhz": self.nv.nvmlDeviceGetMaxClockInfo(self.h, self.nv.NVML_CLOCK_SM)}


def residency(sm, t0, t1):
    """CTAs per SM held at once: (median over SMs of the most at any moment, median of the time average)."""
    import numpy as np
    peaks, means = [], []
    for s in np.unique(sm):
        a, b = t0[sm == s], t1[sm == s]
        ev = np.concatenate([np.stack([a, np.ones_like(a)], 1), np.stack([b, -np.ones_like(b)], 1)])
        ev = ev[np.lexsort((ev[:, 1], ev[:, 0]))]          # an end before a start at the same clock
        peaks.append(int(np.cumsum(ev[:, 1]).max()))
        means.append(float((b - a).sum()) / float(max(b.max() - a.min(), 1)))
    return float(np.median(peaks)), float(np.median(means))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", help="a libregk.so built with -DREGK_PHASE_STAMPS (default: build one now)")
    ap.add_argument("--config", default="config3")
    ap.add_argument("--records", type=int, default=10_000_000)
    ap.add_argument("--steps", type=int, default=6, help="stamped steps (batches rotated); all their CTAs are pooled")
    ap.add_argument("--label", default="")
    ap.add_argument("--out", help="also write the JSON line to this file")
    a = ap.parse_args()

    lib = a.lib
    if not lib:
        lib = build_instrumented(tempfile.mkdtemp(prefix="regk_phases_"))
    os.environ["REGK_LIB"] = os.path.abspath(lib)

    import ctypes as C
    import numpy as np
    import torch
    from registrar_b200 import _native, multigpu, synth

    dev = torch.device("cuda", 0)
    handle = _native.load_library()
    if not hasattr(handle, "regk_phase_stamps"):
        sys.exit("%s was not built with -DREGK_PHASE_STAMPS" % lib)
    handle.regk_phase_stamps.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
    ctx = _native.Context(0)
    n = a.records
    hbs = [synth.generate(a.config, n=n, start=b * n) for b in range(2)]
    ctx.set_types(hbs[0].types)
    cbs = [multigpu.device_batch(hb, dev) for hb in hbs]
    torch.cuda.synchronize()
    ntiles = (n + 127) // 128
    buf = torch.zeros(2 * ntiles * 8, dtype=torch.int64, device=dev)

    for i in range(4):                                     # warm-up, unstamped
        ctx.register_raw(cbs[i % 2][0])
    clock = Clock()
    clock.start()
    rows = {"path": [], "json": []}
    generic = 0
    ctx._check(handle.regk_phase_stamps(ctx._h, C.c_void_p(buf.data_ptr()), ntiles))
    for i in range(a.steps):
        buf.zero_()
        torch.cuda.synchronize()
        clock.active.set()
        r = ctx.register_raw(cbs[i % 2][0])
        clock.active.clear()
        generic = max(generic, int(r.generic_tiles))
        st = buf.view(2, ntiles, 8).cpu().numpy().astype(np.int64)
        for k, name in enumerate(("path", "json")):
            s = st[k]
            rows[name].append(s[(s[:, 0:5] != 0).all(1)])
    ctx._check(handle.regk_phase_stamps(ctx._h, None, 0))
    clock.stop.set()
    mhz = float(np.median(clock.samples)) if clock.samples else float("nan")

    out = {"label": a.label, "config": a.config, "records": n, "steps": a.steps, "generic_tiles": generic,
           "card": clock.card(), "sm_mhz_median": mhz}
    for name in ("path", "json"):
        s = np.concatenate(rows[name])
        ph = {}
        for key, i0, i1 in PHASES[name]:
            us = (s[:, i1] - s[:, i0]) / mhz
            ph[key] = {"median_us": round(float(np.median(us)), 3), "p90_us": round(float(np.percentile(us, 90)), 3)}
        ph["prologue_share"] = round(ph["prologue"]["median_us"] / ph["life"]["median_us"], 3)
        res = [residency(x[:, 7], x[:, 0], x[:, 4]) for x in rows[name]]      # per step: steps are apart in time
        out[name] = {"ctas": int(len(s)), "phases": ph,
                     "resident_ctas_per_sm": {"peak": float(np.median([q[0] for q in res])),
                                              "mean": round(float(np.median([q[1] for q in res])), 2)}}
    ctx.close()
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
