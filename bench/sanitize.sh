#!/bin/bash
# compute-sanitizer passes over the kernel library (SURVEY 5.2).  Runs on ONE GPU; the wgmma /
# TMA kernels are checked with memcheck + synccheck, the element-wise kernels additionally with
# racecheck (racecheck does not model async-proxy (TMA / wgmma) shared-memory traffic).
set -u
# every test tensor its own allocation: with the caching allocator an overrun lands inside a cached
# segment that memcheck counts as valid memory
export PYTORCH_NO_CUDA_MEMORY_CACHING=1
mkdir -p ${OUT:-prof_out}
SAN=/usr/local/cuda/bin/compute-sanitizer
K='gemm_kk and 128-64-64 or gemm_kk and 4096-5-4096 or gemm_mnk and 4096-16-512 or gemm_mnmn_store and 10-4096-5'
K+=' or gemm_mnmn_bf16 and 10-4096-37 or bias_relu and 300-48-64 or conv_fprop and 2-16-16 or conv_wgrad and 2-16-16'
K+=' or conv_dgrad and 2-32-32 or conv0_fused and 2-16-16 or fprop_pool_fused and 2-32-32 or fprop_pool_fused and 4-14-14'
K+=' or maxpool or cross_entropy and 64-3 or adam or bias_grad and 64-3 or head_ce'
for tool in memcheck synccheck; do
  timeout 900 $SAN --tool $tool --error-exitcode 7 python -m pytest tests/test_kernels_gpu.py -q -x -m gpu -k "$K" \
      > ${OUT:-prof_out}/sanitize_$tool.log 2>&1
  echo "== compute-sanitizer $tool exit $?"; grep -E "ERROR SUMMARY|passed|failed" ${OUT:-prof_out}/sanitize_$tool.log | tail -3
done
# the 256-wide conv tiles: fprop, fprop + pool, dgrad (plain / masked / column sum) and wgrad, one small case each
for tool in memcheck synccheck; do
  timeout 900 $SAN --tool $tool --error-exitcode 7 python -m pytest tests/test_wide_tiles_gpu.py -q -x -m gpu \
      -k "exact and 2-28-28-256-256" > ${OUT:-prof_out}/sanitize_wide_$tool.log 2>&1
  echo "== compute-sanitizer $tool (256-wide tiles) exit $?"; grep -E "ERROR SUMMARY|passed|failed" ${OUT:-prof_out}/sanitize_wide_$tool.log | tail -3
done
# one small case of each family of the float64 element-wise tests, under memcheck and racecheck
E='maxpool_fwd_relu_bwd_colsum and 3-16-8 or avgpool_fwd_bwd and 5-64-1 or bias_grad and 37-3-8 or bias_grad and 64-64-64'
E+=' or fc_bias_act_and_dropout and 37-10-0.6 or fc_grad_act and 1-5-True or test_cross_entropy and 7-10 or head_ce and 37-3'
E+=' or adam_steps or sgd_steps and 0.0 or casts and 4099 or nchw_to_nhwc_zero_pads and 1-3-5'
for tool in memcheck racecheck; do
  timeout 900 $SAN --tool $tool --error-exitcode 7 python -m pytest tests/test_elementwise_gpu.py -q -x -m gpu -k "$E" \
      > ${OUT:-prof_out}/sanitize_elementwise_$tool.log 2>&1
  echo "== compute-sanitizer $tool (elementwise) exit $?"
  grep -E "RACECHECK SUMMARY|ERROR SUMMARY|passed|failed" ${OUT:-prof_out}/sanitize_elementwise_$tool.log | tail -3
done
timeout 900 $SAN --tool racecheck --error-exitcode 7 python -m pytest tests/test_kernels_gpu.py -q -x -m gpu \
    -k "maxpool or cross_entropy and 64-3 or bias_grad and 64-3 or adam or head_ce" > ${OUT:-prof_out}/sanitize_racecheck.log 2>&1
echo "== compute-sanitizer racecheck exit $?"; grep -E "RACECHECK SUMMARY|ERROR SUMMARY|passed|failed" ${OUT:-prof_out}/sanitize_racecheck.log | tail -3
