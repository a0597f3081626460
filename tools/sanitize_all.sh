for tool in memcheck racecheck synccheck; do
  echo "== compute-sanitizer --tool $tool"
  timeout 900 compute-sanitizer --tool $tool python tests/sanitize_run.py 2>&1 | tail -4
  timeout 900 compute-sanitizer --tool $tool python tests/sanitize_skip_run.py 2>&1 | tail -4
  timeout 900 compute-sanitizer --tool $tool python tests/sanitize_mkdirp_run.py 2>&1 | tail -4
  timeout 1800 compute-sanitizer --tool $tool python tests/sanitize_prefetch_run.py 2>&1 | tail -4
  timeout 900 compute-sanitizer --tool $tool python tests/sanitize_reconcile_run.py 2>&1 | tail -4
  timeout 900 compute-sanitizer --tool $tool python tests/sanitize_reconcile_owned_run.py 2>&1 | tail -4
  timeout 900 compute-sanitizer --tool $tool python tests/sanitize_replies_run.py 2>&1 | tail -4
done > gpurun_out/r2_sanitizer_new.txt 2>&1
cat gpurun_out/r2_sanitizer_new.txt
