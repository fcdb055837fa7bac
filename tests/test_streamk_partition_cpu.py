"""Property test of the stream-K work partition and partial-tile flag protocol of the GEMM (ops/csrc/gemm_sm90.cu:
`work_range` / `next_work`, the `partner_end` loop of the consumer epilogue, and the host's `per` / grid computation in
`tepd_gemm_bf16` when split_k < 0).

This is a PYTHON MIRROR of that index arithmetic, transcribed by hand -- the device code itself cannot run here.  So a pass
means "the arithmetic as transcribed is sound for these shapes"; a transcription slip would go unnoticed.  What the GPU numerics
checks cover is the real code on about ten shapes (tests/kernel_checks.py::check_gemm2, run twice in a row so a flag left set
would show); what this adds is breadth: thousands of (tiles, k_blocks, CTAs) combinations, including the default-path user of
stream-K (lm_head weight gradient, 128 x 256 tiles, 64 k-blocks, one CTA per SM of an H100).

Why it matters: a CTA whose range starts mid-tile stores a partial tile and raises flag[cta]; the CTA holding k-block 0 of that
tile waits for the flags of the CTAs that follow it inside the tile, sums their partials and RESETS the flags.  A flag that is
raised but never consumed would still be 1 at the next launch and let a finisher read a stale partial tile -- silent corruption
that neither the numerics of a single launch nor compute-sanitizer's racecheck (shared memory only) would show.  The finisher's
wait is deadlock-free only if every CTA of the grid is resident at once (grid <= SMs, one CTA per SM) and the flag-raising unit
is a CTA's first.
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


def partners_of(cta, tile, per, k_blocks, grid):
    """epilogue of a finisher unit: CTAs cta+1 .. partner_end-1"""
    tile_end = (tile + 1) * k_blocks
    end = cta + 1
    while end < grid and end * per < tile_end:
        end += 1
    return list(range(cta + 1, end))


def check(total_tiles, k_blocks, num_sms):
    per, grid = host_partition(total_tiles, k_blocks, num_sms)
    assert grid <= num_sms, "more CTAs than SMs: finishers could wait for CTAs that are not resident"
    units = [units_of(c, per, k_blocks, total_tiles) for c in range(grid)]
    covered = {}
    setters = set()          # CTAs that raise their flag
    consumed = {}            # CTA -> finisher that resets its flag
    for c, seq in enumerate(units):
        for s, (tile, kb0, kb1) in enumerate(seq):
            assert 0 <= kb0 < kb1 <= k_blocks and 0 <= tile < total_tiles, (c, s, tile, kb0, kb1)
            for kb in range(kb0, kb1):
                assert (tile, kb) not in covered, f"(tile {tile}, kb {kb}) done by CTA {covered[(tile, kb)]} and {c}"
                covered[(tile, kb)] = c
            partial = not (kb0 == 0 and kb1 == k_blocks)
            if partial and kb0 > 0:                      # sk_store
                assert s == 0, f"CTA {c}: the flag-raising unit runs at position {s}, not first (deadlock-freedom premise)"
                assert c not in setters
                setters.add(c)
            if partial and kb0 == 0:                     # sk_finish
                ps = partners_of(c, tile, per, k_blocks, grid)
                assert ps, f"CTA {c} holds a head part of tile {tile} but finds no partner"
                pos = kb1
                for j in ps:
                    t2, a, b = units[j][0]
                    # partners continue the tile contiguously, each with its FIRST unit
                    assert t2 == tile and a == pos and a > 0, (c, tile, j, (t2, a, b), pos)
                    pos = b
                    assert j not in consumed, f"flag of CTA {j} reset by CTA {consumed[j]} and {c}"
                    consumed[j] = c
                assert pos == k_blocks, f"tile {tile}: head of CTA {c} + partners end at k-block {pos} of {k_blocks}"
    # everything computed exactly once
    assert len(covered) == total_tiles * k_blocks
    # every raised flag is consumed exactly once, and nothing else is waited on
    assert setters == set(consumed), (sorted(setters - set(consumed)), sorted(set(consumed) - setters))
    return per, grid, len(setters)


def test_lm_head_weight_gradient_shape_on_the_default_path():
    # 50304 x 1024 output in 128 x 256 tiles = 393 x 4 tiles, 4096 tokens = 64 k-blocks, 132 SMs
    per, grid, nflags = check(393 * 4, 64, 132)
    assert grid == 132 and nflags > 0


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


def _fails_somewhere(shapes):
    for sh in shapes:
        try:
            check(*sh)
        except AssertionError:
            return True
    return False


_PROBE = [(t, kb, 132) for t in (48, 64, 100, 393 * 4) for kb in (16, 48, 64)] + [(t, kb, 7) for t in range(1, 30) for kb in (3, 5, 16)]


def test_checker_catches_off_by_one_in_partner_scan(monkeypatch):
    """Self-test: `<=` instead of `<` against tile_end makes a finisher wait for (and reset) a CTA of the NEXT tile."""
    import sys
    mod = sys.modules[__name__]

    def bad(cta, tile, per, k_blocks, grid):
        tile_end = (tile + 1) * k_blocks
        end = cta + 1
        while end < grid and end * per <= tile_end:
            end += 1
        return list(range(cta + 1, end))
    monkeypatch.setattr(mod, "partners_of", bad)
    assert _fails_somewhere(_PROBE)


def test_checker_catches_flag_raising_unit_not_first(monkeypatch):
    """Self-test: if a change of the walk order ever moved the leading partial unit away from position 0, a finisher could wait
    on a CTA that is itself still waiting -- the checker must notice the premise is gone."""
    import sys
    mod = sys.modules[__name__]
    orig = mod.units_of

    def bad_units(cta, per, k_blocks, total_tiles):
        seq = orig(cta, per, k_blocks, total_tiles)
        if len(seq) >= 2 and seq[0][1] > 0:      # swap the first two units
            seq[0], seq[1] = seq[1], seq[0]
        return seq
    monkeypatch.setattr(mod, "units_of", bad_units)
    assert _fails_somewhere(_PROBE)
