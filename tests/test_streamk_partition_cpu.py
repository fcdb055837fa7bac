"""Property test of the stream-K work partition of the GEMM (ops/csrc/gemm_sm90.cu: `work_range` / `next_work` and the
host's `per` / grid computation in `tepd_gemm_bf16` when split_k < 0).

This is a PYTHON MIRROR of that index arithmetic, transcribed by hand -- the device code itself cannot run here.  So a pass
means "the arithmetic as transcribed is sound for these shapes"; a transcription slip would go unnoticed.  The GPU numerics
tests cover the real code on a handful of shapes (tests/test_step_numerics_gpu.py::test_gemm_stream_k_exact,
tests/test_gemm_f32_epilogue_gpu.py); what this adds is breadth: thousands of (tiles, k_blocks, CTAs) combinations, including
the lm_head weight gradient (128 x 256 tiles, 64 k-blocks, one CTA per SM of an H100), which runs stream-K when micro-batch
gradients accumulate into it.

Why it matters: stream-K serves fp32 accumulating outputs only, and every unit adds its partial into the output.  A
(tile, k-block) that no unit covers, or that two units cover, changes the sum silently.
"""
import os
import random

import pytest


def host_partition(total_tiles, k_blocks, num_sms):
    """tepd_gemm_bf16 with split_k < 0: k-block iterations per CTA and number of CTAs launched."""
    iters = total_tiles * k_blocks
    per = (iters + num_sms - 1) // num_sms
    per = max(per, 4)
    grid = (iters + per - 1) // per
    return per, grid


def units_of(cta, per, k_blocks, total_tiles):
    """work_range + repeated next_work for the stream-K case: [(tile, kb0, kb1)] in execution order."""
    total = total_tiles * k_blocks
    c0 = cta * per
    cursor, end = min(c0, total), min(c0 + per, total)
    out = []
    while cursor < end:
        t = cursor // k_blocks
        kb0 = cursor - t * k_blocks
        kb1 = min(k_blocks, kb0 + (end - cursor))
        cursor += kb1 - kb0
        out.append((t, kb0, kb1))
    return out


def check(total_tiles, k_blocks, num_sms):
    per, grid = host_partition(total_tiles, k_blocks, num_sms)
    assert grid <= num_sms, "more CTAs than SMs: the persistent grid would run in more than one wave"
    covered = {}
    split_tiles = set()      # tiles whose k range is shared by more than one unit
    for c in range(grid):
        for s, (tile, kb0, kb1) in enumerate(units_of(c, per, k_blocks, total_tiles)):
            assert 0 <= kb0 < kb1 <= k_blocks and 0 <= tile < total_tiles, (c, s, tile, kb0, kb1)
            for kb in range(kb0, kb1):
                assert (tile, kb) not in covered, f"(tile {tile}, kb {kb}) done by CTA {covered[(tile, kb)]} and {c}"
                covered[(tile, kb)] = c
            if not (kb0 == 0 and kb1 == k_blocks):
                split_tiles.add(tile)
    # everything computed exactly once
    assert len(covered) == total_tiles * k_blocks
    return per, grid, len(split_tiles)


def test_lm_head_weight_gradient_shape_on_the_default_path():
    # 50304 x 1024 output in 128 x 256 tiles = 393 x 4 tiles, 4096 tokens = 64 k-blocks, 132 SMs
    per, grid, nsplit = check(393 * 4, 64, 132)
    assert grid == 132 and nsplit > 0


@pytest.mark.parametrize("pairs", [1, 2, 3, 7, 37, 73, 74, 131, 132])
def test_exhaustive_small_shapes(pairs):
    for tiles in range(1, 41):
        for kb in (1, 2, 3, 4, 5, 7, 8, 16, 17, 64):
            check(tiles, kb, pairs)


def test_random_shapes():
    rng = random.Random(1234)
    for _ in range(4000 if os.environ.get("TEPDIST_TEST_FULL") == "1" else 1200):
        check(rng.randint(1, 1600), rng.randint(1, 96), rng.choice([132, 132, 132, 114, 66, 16, 8]))


def test_transformer_shapes():
    for (m, n, k) in [(4096, 1024, 1024), (4096, 3072, 1024), (4096, 4096, 1024), (4096, 1024, 4096), (4096, 50304, 1024),
                      (1000, 520, 2048), (512, 512, 8192), (384, 520, 200), (3072, 1024, 4096), (1024, 1024, 4096)]:
        tiles = ((m + 127) // 128) * ((n + 255) // 256)
        check(tiles, (k + 63) // 64, 132)
