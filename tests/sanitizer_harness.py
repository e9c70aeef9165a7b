"""Runs a GPU test target under compute-sanitizer; the allocator poisoning the targets and tests use, the body every
target shares (target_main) and the tests' check that a run repeats bit for bit on poisoned memory (assert_repeatable).

A target is a small script that prints a marker line when it finishes and, with G2PC_TARGET_OUT=<file.npz>, saves every
output of its run there.  Where compute-sanitizer is missing or does not support the GPU, the target runs without it and
the check is made from its outputs, which must match bit for bit:
  memcheck   three runs whose allocator memory starts filled with 0x00, 0xff and 0x5a (G2PC_TARGET_POISON), with
             CUDA_LAUNCH_BLOCKING=1: an illegal address fails the launch that made it, and a read of memory nobody wrote
             makes the outputs depend on the fill byte;
  racecheck  the same three poisoned runs, or, with repeat_racecheck, three identical runs: a race makes them disagree."""
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

from util import same

DEV = "cuda:0"


def poison_allocator(byte, large_bytes=64 << 20, large_blocks=4):
    """Fill and release blocks of both pools of PyTorch's caching allocator (it keeps them cached), so memory a kernel
    reads without writing it first holds `byte`.  First every free block the allocator still caches: empty_cache keeps
    the segments that hold a live tensor (say one cached by an earlier test), and a request would be served from their
    free tails before any new block.  Then fresh segments: small pool, blocks of <= 1 MB carved from 2 MB segments;
    large pool, split blocks of the large_blocks segments of large_bytes.  A block served by a fresh cudaMalloc after
    this is not poisoned."""
    import torch
    torch.cuda.empty_cache()
    stream = torch.cuda.current_stream(DEV).cuda_stream
    free = sorted((seg["segment_type"] == "large", b["size"]) for seg in torch.cuda.memory_snapshot()
                  if seg.get("device", 0) == torch.device(DEV).index and seg["stream"] == stream
                  for b in seg["blocks"] if b["state"] == "inactive")
    # A request of <= 1 MB is served from the small pool, a larger one from the large pool, each from the smallest free
    # block that fits: so small-pool blocks are claimed in pieces of <= 1 MB, and large-pool blocks (all > 1 MB) whole,
    # smallest first, each by a request of its own size.
    sizes = []
    for large, nbytes in free:
        sizes += [nbytes] if large else [1 << 20] * (nbytes >> 20) + [nbytes & ((1 << 20) - 1)]
    tails = [torch.empty((n,), dtype=torch.uint8, device=DEV).fill_(byte) for n in sizes if n]
    small = [torch.full((1 << 20,), byte, dtype=torch.uint8, device=DEV) for _ in range(64)]
    large = [torch.full((large_bytes,), byte, dtype=torch.uint8, device=DEV) for _ in range(large_blocks)]
    torch.cuda.synchronize()
    del tails, small, large
    for nbytes in (4096, 8 << 20):  # later blocks of both pools really start out filled
        probe = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
        assert bool((probe == byte).all()), f"allocator memory not poisoned ({nbytes} B block)"
        del probe


def assert_repeatable(run, **poison_kwargs):
    """Two runs of run() (a list of host outputs: arrays, or plain values such as cycle counts), then a third on
    allocator memory filled by poison_allocator(**poison_kwargs); all three must agree bit for bit.  Returns the first
    run's outputs."""
    runs = [run() for _ in range(2)]
    poison_allocator(**poison_kwargs)
    runs.append(run())
    for r in runs[1:]:
        assert len(r) == len(runs[0])
        for a, b in zip(runs[0], r):
            assert same(a, b) if isinstance(a, np.ndarray) else a == b
    return runs[0]


def target_main(marker, run, **poison_kwargs):
    """The body of a target script: poisons the allocator with poison_allocator(G2PC_TARGET_POISON, **poison_kwargs)
    when that variable is set, calls run() -> (dict of output tensors, values to print), saves the outputs to
    G2PC_TARGET_OUT when that is set, and prints the marker line with the values."""
    import torch
    if os.environ.get("G2PC_TARGET_POISON") is not None:
        poison_allocator(int(os.environ["G2PC_TARGET_POISON"], 0), **poison_kwargs)
    outputs, values = run()
    torch.cuda.synchronize()
    if os.environ.get("G2PC_TARGET_OUT"):
        np.savez(os.environ["G2PC_TARGET_OUT"], **{k: v.detach().cpu().numpy() for k, v in outputs.items()})
    print(marker, *values)


def _sanitizer():
    return shutil.which("compute-sanitizer") or (
        "/usr/local/cuda/bin/compute-sanitizer" if os.path.exists("/usr/local/cuda/bin/compute-sanitizer") else None)


def _run_target(target, marker, timeout, env_extra, out):
    env = dict(os.environ, G2PC_TARGET_OUT=str(out), **env_extra)
    r = subprocess.run([sys.executable, target], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env,
                       timeout=timeout)
    assert r.returncode == 0 and marker in r.stdout, r.stdout[-3000:]
    with np.load(out) as z:
        return {k: z[k] for k in z.files}


def _check_from_outputs(target, marker, tool, timeout, tmp_path, repeat_racecheck):
    if tool == "racecheck" and repeat_racecheck:
        runs = [_run_target(target, marker, timeout, {"G2PC_TARGET_POISON": "0x00"}, tmp_path / f"repeat_{i}.npz")
                for i in range(3)]
    else:
        runs = [_run_target(target, marker, timeout, {"G2PC_TARGET_POISON": b, "CUDA_LAUNCH_BLOCKING": "1"},
                            tmp_path / f"fill_{b}.npz") for b in ("0x00", "0xff", "0x5a")]
    first = runs[0]
    for i, other in enumerate(runs[1:], 1):
        assert sorted(other) == sorted(first)
        for k in first:
            assert other[k].dtype == first[k].dtype and other[k].shape == first[k].shape, (tool, i, k)
            assert other[k].tobytes() == first[k].tobytes(), f"{tool}: run {i} differs from run 0 in {k}"
    return first


def check_target(target, marker, tool, tmp_path, timeout, repeat_racecheck=False):
    """Runs `target` under compute-sanitizer's `tool` (memcheck or racecheck) and asserts a clean report, or, where the
    tool cannot run, makes the check from the outputs of three runs.  Returns the outputs of the first of those runs,
    or None when the sanitizer ran."""
    exe = _sanitizer()
    if exe is None:
        return _check_from_outputs(target, marker, tool, timeout, tmp_path, repeat_racecheck)
    # only the library's own kernels (all live in anonymous namespaces of libg2pc.so) are instrumented
    # --report-api-errors no: the CUDA runtime's lazy module loading probes kernels with cuKernelGetFunction and handles
    # the INVALID_HANDLE return itself; memcheck would otherwise count that host-API return code as an error
    cmd = [exe, "--tool", tool, "--kernel-name", "kns=_GLOBAL__N_"] + \
          (["--report-api-errors", "no"] if tool == "memcheck" else []) + ["--print-limit", "5", sys.executable, target]
    try:
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=timeout)
    except subprocess.TimeoutExpired:
        pytest.skip(f"compute-sanitizer run exceeded {timeout // 60} minutes on this box")
    if "Error: Device not supported" in r.stdout:
        return _check_from_outputs(target, marker, tool, timeout, tmp_path, repeat_racecheck)
    tail = r.stdout[-3000:]
    assert marker in r.stdout, tail
    if tool == "racecheck":
        assert "RACECHECK SUMMARY: 0 hazards displayed (0 errors, 0 warnings)" in r.stdout, tail
    else:
        assert "ERROR SUMMARY: 0 errors" in r.stdout, tail
    return None
