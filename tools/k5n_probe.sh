#!/bin/bash
# development aid: per-kernel times of the lazy pipeline-B update (ncu launch list) + whole-step sweep at the points it matters
ll() { ncu --metrics gpu__time_duration.sum --clock-control none -c 24 --csv python tools/spec_probe.py --one $1 2>/dev/null | grep -E "spectrum|k5_need|epilogue|transpose" | sed -E "s/.*glb::([a-z0-9_]+).*\"ns\",\"([0-9]+)\"/\1 \2/" | tail -4; }
python -m pytest tests/test_gpu_spectrum.py tests/test_gpu_optional.py tests/test_gpu_masked.py tests/test_llvmpipe_golden.py -m gpu -q 2>&1 | tail -8
for S in 1 2 4; do echo "== launches 8192 K5N_S=$S"; GLAVA_B200_K5N_S=$S ll 8192; done
echo "== launches 16384"; ll 16384
echo "== launches 4096 3k"; GLAVA_B200_K5_SPLIT=1 ll 4096
echo "== sweep default"; python tools/sweep_configs.py bars:4096:1920x1080 bars:8192:1280x720 bars:8192:1920x1080 bars:16384:1280x720 bars:16384:1920x1080 radial:8192:3840x2160 2>&1 | cut -c1-200
echo "== sweep 4096 3k"; GLAVA_B200_K5_SPLIT=1 python tools/sweep_configs.py bars:4096:1920x1080 bars:4096:1280x720 bars:2048:1280x720 2>&1 | cut -c1-200
echo "== sweep 4096 3k oop128"; GLAVA_B200_K5_SPLIT=1 GLAVA_B200_SPEC_OOP=1 GLAVA_B200_SPEC_T=128 python tools/sweep_configs.py bars:4096:1920x1080 bars:4096:1280x720 bars:2048:1280x720 2>&1 | cut -c1-200
echo "== circle tests"; python -m pytest tests/test_gpu_raster.py tests/test_glsl_golden.py tests/test_llvmpipe_golden.py -m gpu -q -k "circle or raster" 2>&1 | tail -4
echo "== circle sweep (tile cull off / on)"; python tools/sweep_configs.py circle:4096:1920x1080 2>&1 | cut -c1-330; GLAVA_B200_CTILE=1 python tools/sweep_configs.py circle:4096:1920x1080 2>&1 | cut -c1-330
