"""SURVEY §5: run the hot path under compute-sanitizer (memcheck + racecheck) on a tiny scene.

Where compute-sanitizer is missing or does not support the GPU, the same target runs without it and the two checks are
made from its outputs, which are deterministic (integer atomics only, order-independent merges):
  memcheck   three runs whose allocator memory starts filled with 0x00, 0xff and 0x5a, with CUDA_LAUNCH_BLOCKING=1: an
             illegal address fails the launch that made it, and a read of memory the pipeline never wrote (uninitialised,
             or past the end of a buffer into pool memory) makes the outputs depend on the fill byte;
  racecheck  three identical runs with the two frames in flight: a race in the staging buffers, the s_best merge, the
             multisplit bit matrix or between the frame streams makes them disagree.
Every output (per-Gaussian accumulators of both back-ends, cull index, point cloud) must match bit for bit."""
import os

import pytest

from sanitizer_harness import check_target

pytestmark = pytest.mark.gpu
TARGET = os.path.join(os.path.dirname(os.path.abspath(__file__)), "sanitizer_target.py")


@pytest.mark.parametrize("tool", ["memcheck", "racecheck"])
def test_hot_path_is_clean_under_compute_sanitizer(lib, tool, tmp_path):
    first = check_target(TARGET, "SANITIZER_TARGET_OK", tool, tmp_path, timeout=900, repeat_racecheck=True)
    if first is not None:
        assert len(first) >= 10 and first["points"].shape[0] > 0
