#!/bin/bash
# compute-sanitizer evidence (SURVEY §5): memcheck + racecheck + synccheck over the smoke invocation (forward + fused
# scheduler step: conv_tc / conv_in / conv_out / attention / temb kernels) and memcheck + racecheck over one small backward
# (backward / wgrad_tc / bwd kernels) and the Mel codec.  Each run logs to sanitizer_<tool>_<what>_<tag>.log in the
# output directory below; the summaries are copied to profiles/.
# usage (on the GPU box): tools/sanitize.sh [tag]
tag=${1:-r02}
mkdir -p gpurun_out
CS=/usr/local/cuda/bin/compute-sanitizer
for tool in memcheck racecheck synccheck; do
  timeout 600 $CS --tool $tool --print-limit 20 --log-file gpurun_out/sanitizer_${tool}_smoke_${tag}.log \
    python -c "import __graft_entry__ as g; g.smoke()" > gpurun_out/sanitizer_${tool}_smoke_${tag}.out 2>&1
  echo "$tool smoke: exit $?"
  tail -3 gpurun_out/sanitizer_${tool}_smoke_${tag}.log
done
# the backward cases: the plain backward, and one with gradient checkpointing (it re-runs forward ops into shared buffers)
for tool in memcheck racecheck; do
  timeout 900 $CS --tool $tool --print-limit 20 --log-file gpurun_out/sanitizer_${tool}_bwd_${tag}.log \
    python -m pytest tests/test_gpu_train.py tests/test_gpu_checkpointing.py -x -q -m gpu \
    -k "test_unet_backward_matches_autograd or (test_checkpointed_training_matches_plain and published)" \
    > gpurun_out/sanitizer_${tool}_bwd_${tag}.out 2>&1
  echo "$tool backward: exit $?"
  tail -3 gpurun_out/sanitizer_${tool}_bwd_${tag}.log
done
for tool in memcheck racecheck; do
  timeout 600 $CS --tool $tool --print-limit 20 --log-file gpurun_out/sanitizer_${tool}_mel_${tag}.log \
    python -m pytest tests/test_gpu_mel.py -x -q -m gpu > gpurun_out/sanitizer_${tool}_mel_${tag}.out 2>&1
  echo "$tool mel: exit $?"
  tail -3 gpurun_out/sanitizer_${tool}_mel_${tag}.log
done
# racecheck again WITHOUT conv_tc_kernel: its only reports are write/write pairs between the TMA bulk copy that fills an
# activation stage and the transform warps that rewrite it in place (ordered by the stage's full / empty mbarriers, which
# the tool does not follow for async-proxy copies) and they exhaust the hazard limit before any other kernel is looked at
for what in smoke bwd; do
  if [ $what = smoke ]; then cmd=(python -c "import __graft_entry__ as g; g.smoke()");
  else cmd=(python -m pytest tests/test_gpu_train.py -x -q -m gpu -k test_unet_backward_matches_autograd); fi
  timeout 900 $CS --tool racecheck --kernel-name-exclude kns=conv_tc_kernel --print-limit 20 \
    --log-file gpurun_out/sanitizer_racecheck_noconvtc_${what}_${tag}.log "${cmd[@]}" > gpurun_out/sanitizer_racecheck_noconvtc_${what}_${tag}.out 2>&1
  echo "racecheck (all kernels but conv_tc) $what: exit $?"
  tail -3 gpurun_out/sanitizer_racecheck_noconvtc_${what}_${tag}.log
done
