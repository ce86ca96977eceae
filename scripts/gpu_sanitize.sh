#!/bin/bash
# compute-sanitizer passes over smoke() (one tiny forward through every kernel of the hot path)
# and over a single causal streaming step.  Usage: gpurun -- bash scripts/gpu_sanitize.sh
cd "$(dirname "$0")/.." || exit 1
mkdir -p gpurun_out
for tool in memcheck racecheck synccheck; do
  timeout 900 compute-sanitizer --tool $tool --print-limit 20 \
      python -c "import __graft_entry__ as g; g.smoke(); g.smoke_stream()" \
      > gpurun_out/sanitizer_$tool.log 2>&1
  echo "sanitizer $tool rc=$? $(grep -E 'ERROR SUMMARY|RACECHECK SUMMARY' gpurun_out/sanitizer_$tool.log | tail -1)"
done
# then the YUV 4:2:0 readers (stem loader, ingest taps, conversion kernel) on pitched, cropped
# frames; the sanitizer's findings and summary go to stdout
for tool in memcheck racecheck; do
  timeout 1800 compute-sanitizer --tool $tool --print-limit 20 \
      python -m pytest -q -m gpu -p no:cacheprovider tests/test_yuv_gpu.py -k "not every_triple" \
      2>&1 | grep -E '^=========|passed|failed' | tail -n 25
  echo "sanitizer yuv $tool rc=${PIPESTATUS[0]}"
done
# the general YUV reader (16-bit, packed 4:2:2 and 4:4:4 layouts) through the same three kernels
timeout 1800 compute-sanitizer --tool memcheck --print-limit 20 \
    python -m pytest -q -m gpu -p no:cacheprovider tests/test_yuv_formats_gpu.py \
    -k "random_samples or same_bytes or side_stream or feature_grids" \
    2>&1 | grep -E '^=========|passed|failed' | tail -n 25
echo "sanitizer yuv_formats memcheck rc=${PIPESTATUS[0]}"
# then the backbone's memory-bound kernels one at a time, with NaN guards around every output
# (stem conv, instance norm, im2col, layer norm, L2 norm, resize)
timeout 1800 compute-sanitizer --tool memcheck --print-limit 20 \
    python -m pytest -q -m gpu -p no:cacheprovider tests/test_backbone_ops_gpu.py -k "not backbone_vs and not frame_chunks" \
    2>&1 | grep -E '^=========|passed|failed' | tail -n 25
echo "sanitizer backbone_ops memcheck rc=${PIPESTATUS[0]}"
# then the refinement kernels one at a time (local correlation, pooling, track update, the mixer's
# depthwise block), leaving out the production-shape cases
timeout 1800 compute-sanitizer --tool memcheck --print-limit 20 \
    python -m pytest -q -m gpu -p no:cacheprovider tests/test_refine_ops_gpu.py \
    -k "not production_shape and not streaming_shape and not clip_shape and not pl1_1024 and not n1001 and not n801 and not n700" \
    2>&1 | grep -E '^=========|passed|failed' | tail -n 25
echo "sanitizer refine_ops memcheck rc=${PIPESTATUS[0]}"
# then every GEMM epilogue path (whole-tile and general epilogues, split-K reduction, halo
# convolution, SIMT) and tapir_split_planes, with NaN-filled padding around every output
timeout 1800 compute-sanitizer --tool memcheck --print-limit 20 \
    python -m pytest -q -m gpu -p no:cacheprovider tests/test_gemm_exact_gpu.py \
    2>&1 | grep -E '^=========|passed|failed' | tail -n 25
echo "sanitizer gemm_exact memcheck rc=${PIPESTATUS[0]}"
# then the Lanczos resize (both passes, one axis, identity, 1-pixel sides, bad arguments); the
# readers and the model runs of the evaluation tests are left out
timeout 1800 compute-sanitizer --tool memcheck --print-limit 20 \
    python -m pytest -q -m gpu -p no:cacheprovider tests/test_tapvid_gpu.py -k "not evaluate and not readers" \
    2>&1 | grep -E '^=========|passed|failed' | tail -n 25
echo "sanitizer tapvid memcheck rc=${PIPESTATUS[0]}"
# then the streams of different frame sizes: the multi-frame ingest (uint8, pitched, NV12 / I420
# windows, more frames than one launch), the per-clip track update and the mixed-size tracker
timeout 1800 compute-sanitizer --tool memcheck --print-limit 20 \
    python -m pytest -q -m gpu -p no:cacheprovider tests/test_tracker_sizes_gpu.py \
    -k "not golden_and_eager and not isolated" \
    2>&1 | grep -E '^=========|passed|failed' | tail -n 25
echo "sanitizer sizes memcheck rc=${PIPESTATUS[0]}"
# then AJ_RD's event kernel (fixture cases, random clips up to 300 x 256, the maximal-event track
# at T = 65536, graph replay); the largest clips and the model runs of evaluate are left out
timeout 1800 compute-sanitizer --tool memcheck --print-limit 20 \
    python -m pytest -q -m gpu -p no:cacheprovider tests/test_redetection_gpu.py \
    -k "not evaluate and not 1500" \
    2>&1 | grep -E '^=========|passed|failed' | tail -n 25
echo "sanitizer redetection memcheck rc=${PIPESTATUS[0]}"
# then the per-clip point-count path: the grouped cost-volume GEMM on its designed maps (tail
# guard past the workspace), the ragged stage A, local correlation and track update against
# per-clip calls and the float64 references, and estimate_trajectories over more than 64 clips;
# the 65535-query call and the 70-stream tracker are left out
timeout 1800 compute-sanitizer --tool memcheck --print-limit 20 \
    python -m pytest -q -m gpu -p no:cacheprovider tests/test_plane_pairs_gpu.py tests/test_stream_points_gpu.py \
    tests/test_refine_ops_gpu.py \
    -k "(cost_volume_pairs or ragged or points_per_clip or more_than_64) and not query_limit and not 70_streams" \
    2>&1 | grep -E '^=========|passed|failed' | tail -n 25
echo "sanitizer ragged memcheck rc=${PIPESTATUS[0]}"
# then the point edits of the online tracker: tapir_sample_query_rows on sentinel rows (one and
# per-clip sizes, 1 and 4 levels, out-of-range requests, graph replay) and the one-stream edited
# tracker; the multi-stream trackers are left out
timeout 1800 compute-sanitizer --tool memcheck --print-limit 20 \
    python -m pytest -q -m gpu -p no:cacheprovider tests/test_stream_edit_gpu.py \
    -k "sample_query_rows or retarget_equals" \
    2>&1 | grep -E '^=========|passed|failed' | tail -n 25
echo "sanitizer stream_edit memcheck rc=${PIPESTATUS[0]}"
