#!/usr/bin/env bash
# compute-sanitizer pass over one tiny invocation of every kernel family (slow: the shapes are kept tiny).
# usage: scripts/sanitize.sh [memcheck|racecheck|synccheck] [log directory, default: a new temporary directory]
tool="${1:-memcheck}"
out="${2:-$(mktemp -d)}"
mkdir -p "$out"
timeout 900 compute-sanitizer --tool "$tool" --error-exitcode 9 --print-limit 20 \
  python -m pytest tests/test_gpu_model.py -x -q -m gpu -k "test_bf16_loss_and_grad_vs_oracle or test_fp32_loss_and_grad_match_oracle" \
  -p no:cacheprovider > "$out/sanitize_${tool}_model.log" 2>&1
echo "model: exit $? : $(grep -E 'ERROR SUMMARY|passed|failed' "$out/sanitize_${tool}_model.log" | tail -n 2 | tr '\n' ' ')"
timeout 900 compute-sanitizer --tool "$tool" --error-exitcode 9 --print-limit 20 \
  python -m pytest tests/test_gpu_decode.py -x -q -m gpu -k "test_persistent_logits_match_oracle_forward" \
  -p no:cacheprovider > "$out/sanitize_${tool}_decode.log" 2>&1
echo "decode: exit $? : $(grep -E 'ERROR SUMMARY|passed|failed' "$out/sanitize_${tool}_decode.log" | tail -n 2 | tr '\n' ' ')"
# the standard sampler at 1, 2 and 24 rows (the BT 1, 8 and 32 kernels): shared-memory filter, Philox noise, the EOS
# counter and the early exit (every row of the 24 ends)
timeout 900 compute-sanitizer --tool "$tool" --error-exitcode 9 --print-limit 20 \
  python -m pytest tests/test_gpu_generate.py -x -q -m gpu -k "test_reference_sampler_unaffected_by_generate or test_eos_ends_sequences_and_the_launch" \
  -p no:cacheprovider > "$out/sanitize_${tool}_generate.log" 2>&1
echo "generate: exit $? : $(grep -E 'ERROR SUMMARY|passed|failed' "$out/sanitize_${tool}_generate.log" | tail -n 2 | tr '\n' ' ')"
# the constrained sampler at 1, 2 and 24 rows: presence flags in the q half, the bias, the minimum length and the early exit
timeout 900 compute-sanitizer --tool "$tool" --error-exitcode 9 --print-limit 20 \
  python -m pytest tests/test_gpu_generate_constraints.py -x -q -m gpu -k "test_reference_sampler_after_constrained_generate or test_min_length_binds_at_24_rows" \
  -p no:cacheprovider > "$out/sanitize_${tool}_constraints.log" 2>&1
echo "constraints: exit $? : $(grep -E 'ERROR SUMMARY|passed|failed' "$out/sanitize_${tool}_constraints.log" | tail -n 2 | tr '\n' ' ')"
# forward prefill: the cache scatter from fp32 and bf16 forwards into 1 and 24 decoder rows, and the decode launch after it
timeout 900 compute-sanitizer --tool "$tool" --error-exitcode 9 --print-limit 20 \
  python -m pytest tests/test_gpu_generate_prefill.py -x -q -m gpu -k "test_scatter_at_1_and_24_rows" \
  -p no:cacheprovider > "$out/sanitize_${tool}_prefill.log" 2>&1
echo "prefill: exit $? : $(grep -E 'ERROR SUMMARY|passed|failed' "$out/sanitize_${tool}_prefill.log" | tail -n 2 | tr '\n' ' ')"
# kernels the tiny model configs do not reach: many-tile / tail GEMMs (all epilogues), wgmma attention, streaming LN backward
timeout 1200 compute-sanitizer --tool "$tool" --error-exitcode 9 --print-limit 20 \
  python -m pytest tests/test_gpu_gemm_tc.py tests/test_gpu_attn_tc.py tests/test_gpu_elementwise.py -x -q -m gpu \
  -k "many_tiles or column_tail or attn_tc or stream_path" -p no:cacheprovider > "$out/sanitize_${tool}_kernels.log" 2>&1
echo "kernels: exit $? : $(grep -E 'ERROR SUMMARY|passed|failed' "$out/sanitize_${tool}_kernels.log" | tail -n 2 | tr '\n' ' ')"
echo "logs in $out"
