"""TEST INFRASTRUCTURE: one pass over the exact-size device batches of tests/test_device_route_gpu.py, the batch queue,
and the long-type table of tests/test_type_table_gpu.py, as a plain run for compute-sanitizer: every input array is
its own exact-size allocation, so memcheck flags any read past a caller's array.  Run on the GPU box:
    compute-sanitizer --tool memcheck python tests/sanitize_device_types_run.py"""
import ctypes as C
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from registrar_b200 import _native
import test_device_route_gpu as dr
import test_type_table_gpu as tt

# the emulation library (only its emul_build_blob is used here), built apart from the test suite's cached copy
so = os.path.join(tempfile.mkdtemp(prefix="regk_sanitize_"), "libregemul.so")
subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-unknown-pragmas", "-o", so,
                       os.path.join(ROOT, "tests", "emul", "emul.cpp")])
emul = C.CDLL(so)
shutil.rmtree(os.path.dirname(so))
emul.emul_build_blob.restype = C.c_int

ctx = _native.Context(0)
for case in ("n=1", "n=129", "n=4097", "alias", "host_off", "ports_off_null", "ports_present", "empty_labels"):
    for in_dev, out_dev in dr.ROUTES:
        dr.check_route(ctx, dr.route_case(case), in_dev, out_dev)
dr.test_queue_batch_by_batch(ctx)
dr.test_queue_out_of_domain_batch(ctx)
tt.test_long_type_goes_generic_tile_by_tile(ctx, emul)
ctx.close()
print("sanitize_device_types_run ok")
