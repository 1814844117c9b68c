#!/usr/bin/env bash
# Run ON THE GPU BOX: compute-sanitizer over small parity tests (memcheck / racecheck / synccheck / initcheck).
# Summaries -> gpurun_out/sanitizer_<tool>_r02.log ; tools/summarise_sanitizer.py writes profiles/sanitizer_r02.md
mkdir -p gpurun_out
CS=/usr/local/cuda/bin/compute-sanitizer
SMALL_MLP='test_dense_layer and (128-32-16 or 300-64-64 or 131-48-80 or 256-32-16 or 1024-64-32 or 160-384-128 or 4144-64-128) or test_fp_first or (test_factored_sa_first_layer_kernels and (1-512-100 or 3-700-129)) or test_factored_fp_first_layer_kernel or (test_factored_fp_layer_channel_major_output and 1-96-40)'
SMALL_MS='(test_fit_matches_reference_golden and (tight or two or pair_far or single or outl10)) or (test_pruned_density_equals_brute_force and (two or coincident or tiny_bw))'
run() { tool=$1; shift; tag=$1; shift
  timeout 1500 $CS --tool $tool --print-limit 20 --launch-timeout 0 "$@" > gpurun_out/sanitizer_${tool}_${tag}_r02.log 2>&1
  echo "== $tool $tag: $(grep -E 'ERROR SUMMARY|RACECHECK SUMMARY|passed|failed' gpurun_out/sanitizer_${tool}_${tag}_r02.log | tail -3 | tr '\n' ' ')"; }
run memcheck mlp python -m pytest tests/test_mlp_gpu.py -q -m gpu -x -k "$SMALL_MLP"
run memcheck ms python -m pytest tests/test_meanshift_gpu.py tests/test_poses_gpu.py tests/test_metrics_gpu.py -q -m gpu -x -k "$SMALL_MS or test_cal_frame_poses_lm or test_best_fit or test_add_adds or test_seg_argmax"
run memcheck pn2 python -m pytest tests/test_pn2_gpu.py -q -m gpu -x -k "three_nn or ball_query or fps_small or gather or interpolate or slab"
run racecheck mlp python -m pytest tests/test_mlp_gpu.py -q -m gpu -x -k "$SMALL_MLP"
run racecheck ms python -m pytest tests/test_meanshift_gpu.py -q -m gpu -x -k "$SMALL_MS"
run synccheck mlp python -m pytest tests/test_mlp_gpu.py -q -m gpu -x -k "$SMALL_MLP"
run synccheck ms python -m pytest tests/test_meanshift_gpu.py -q -m gpu -x -k "$SMALL_MS"
run initcheck ms python -m pytest tests/test_meanshift_gpu.py -q -m gpu -x -k "$SMALL_MS"
ls -la gpurun_out | grep sanitizer
