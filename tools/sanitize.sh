#!/bin/bash
# usage: tools/sanitize.sh   — compute-sanitizer memcheck / racecheck / synccheck over small parity runs of every kernel
# (warp-per-log incl. phase barriers and deferral, admission, patch stream, output packing, both JSON renders, the run / compact
# expansion and adopted device records, the output scan past 2^20 logs, the append splice, the patch window; the c2 case runs the 8-warp team
# kernel).  Needs a GPU and build(); prints a summary per tool and writes nothing.
cd "$(dirname "$0")/.." || exit 1
SEL="kats_through_engine or quirks or mark_boundary_inserted_later or q4_concurrent or dense_surviving or admission_statuses or patch_kats_on_the_device or (fuzz_logs and (0 or 1)) or (generated_workloads_match_oracle and c2-24-2500) or (deferral_on_the_named_side and (comments or overflow or runs-12)) or status_matrix or find_matches_oracle_on_fuzz_sessions or resolve_cursor_kats or find_edge_cases or (each_case_alone and (noncausal or q4 or q3 or q2 or elements)) or failed_logs_are_not_computed or kats_render_on_the_device or unicode_corpus_renders or render_edge_cases or patch_kats_render_on_the_device or unicode_corpus_renders_patches or render_patches_edge_cases or failed_logs_render_patches or (every_form_matches_the_oracle and (kats or status)) or more_than_2_pow_20_logs or (append_after_every_form and (kats or sparse)) or chained_appends or cross_routes or status_corpus_through or refusals_leave or state_rules or (append_then_window and (kats or shared-arrival) and plain)"
for tool in memcheck racecheck synccheck; do
  echo "== $tool"
  timeout 1500 compute-sanitizer --tool $tool --print-limit 5 python -m pytest tests/test_gpu_parity.py tests/test_gpu_round2.py tests/test_gpu_admission.py tests/test_gpu_patches.py tests/test_gpu_workloads.py tests/test_gpu_routes.py tests/test_gpu_find_elements.py tests/test_gpu_patch_bounds.py tests/test_gpu_render_json.py tests/test_gpu_render_patches_json.py tests/test_gpu_wire_forms.py tests/test_gpu_append.py tests/test_gpu_patch_window.py -m gpu -x -q -p no:cacheprovider -k "$SEL" 2>&1 | grep -vE "^=========\s+(at|by|Host Frame|Device Frame|in )|^=========\s*$" | tail -14
done
