#!/bin/bash
# Runs the GPU test tiers in separate processes (a device-side trap poisons its process only)
# and leaves logs + a JSON report in gpurun_out/.  Usage: gpurun -- bash scripts/gpu_ci.sh [tiers]
cd "$(dirname "$0")/.." || exit 1
mkdir -p gpurun_out
TIERS=${*:-"gemm_simt gemm_tc pairs stages_simt stages_tc e2e_simt e2e_tc"}
nvidia-smi --query-gpu=name,clocks.sm,clocks.max.sm,memory.total --format=csv > gpurun_out/gpu_info.txt 2>&1
rc=0
run() {  # name, env, pytest args...
  local name=$1; shift
  local envs=$1; shift
  echo "=== tier $name"
  env $envs timeout 1500 python -m pytest "$@" -q -m gpu --timeout 300 --durations=15 -p no:cacheprovider \
      > "gpurun_out/$name.log" 2>&1
  local r=$?
  tail -n 25 "gpurun_out/$name.log"
  echo "=== tier $name exit $r"
  [ $r -ne 0 ] && rc=1
}
for t in $TIERS; do
  case $t in
    gemm_simt)   run gemm_simt "X=1" tests/test_gemm_gpu.py tests/test_gemm_variants_gpu.py tests/test_gemm_exact_gpu.py -k simt ;;
    gemm_tc)     run gemm_tc "X=1" tests/test_gemm_gpu.py tests/test_gemm_variants_gpu.py tests/test_gemm_schedule_gpu.py tests/test_gemm_exact_gpu.py -k tc ;;
    pairs)       run pairs "X=1" tests/test_plane_pairs_gpu.py ;;
    stages_simt) run stages_simt "TAPIR_B200_GEMM=simt" tests/test_stages_gpu.py tests/test_batched_gpu.py tests/test_stage_a_gpu.py tests/test_backbone_ops_gpu.py tests/test_refine_ops_gpu.py ;;
    stages_tc)   run stages_tc "X=1" tests/test_stages_gpu.py tests/test_batched_gpu.py tests/test_stage_a_gpu.py tests/test_backbone_ops_gpu.py tests/test_refine_ops_gpu.py ;;
    e2e_simt)    run e2e_simt "TAPIR_B200_GEMM=simt" tests/test_end_to_end_gpu.py ;;
    e2e_tc)      run e2e_tc "X=1" tests/test_end_to_end_gpu.py ;;
    props)       run props "X=1" tests/test_properties_gpu.py tests/test_batched_gpu.py ;;
    io)          run io "X=1" tests/test_io_gpu.py ;;
    yuv)         run yuv "X=1" tests/test_yuv_gpu.py ;;
    yuv_formats) run yuv_formats "X=1" tests/test_yuv_formats_gpu.py ;;
    reader)      run reader "X=1" tests/test_windowed_gpu.py tests/test_video_reader_gpu.py ;;
    bulk)        run bulk "X=1" tests/test_bulk_gpu.py ;;
    eval)        run eval "X=1" tests/test_tapvid_gpu.py tests/test_redetection_gpu.py ;;
    sizes)       run sizes "X=1" tests/test_tracker_sizes_gpu.py ;;
    points)      run points "X=1" tests/test_stream_points_gpu.py tests/test_refine_ops_gpu.py::test_local_corr_ragged \
                     tests/test_refine_ops_gpu.py::test_refine_update_bit_exact ;;
    no_halo)     run no_halo "TAPIR_B200_CONV_HALO=0" tests/test_gemm_gpu.py tests/test_gemm_variants_gpu.py tests/test_gemm_exact_gpu.py tests/test_stages_gpu.py tests/test_end_to_end_gpu.py ;;
    all)         run all "X=1" tests ;;
  esac
done
exit $rc
