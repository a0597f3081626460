"""TEST INFRASTRUCTURE: the cases of tests/test_lookahead_prefetch.py as one plain run for compute-sanitizer
(memcheck / racecheck / synccheck): batches longer than one wave on every route, and corrupt offsets in tiles that
other CTAs size their L2 prefetches from.  Run on the GPU box:
    compute-sanitizer --tool memcheck python tests/sanitize_prefetch_run.py"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from registrar_b200 import _native
import test_lookahead_prefetch as t

ctx = _native.Context(0)
t.test_longer_than_a_wave(ctx, "config3", 400_000)
t.test_longer_than_a_wave(ctx, "config5", 300_000)
t.test_device_resident_batch(ctx)
t.test_variable_hostnames_and_alias(ctx)
t.test_pipelined_host_route(ctx)
t.test_skip_mode_long_batch(ctx)
for case in ("dom_decreasing", "dom_past_end", "dom_tile_boundary", "addr_decreasing", "addr_past_end",
             "addr_tile_boundary", "ports_past_end", "ports_tile_boundary"):
    t.test_corrupt_offsets_in_a_lookahead_tile(ctx, case)
ctx.close()
print("sanitize_prefetch_run ok")
