"""SASS budget of the FAST cell kernel's passes (tools/fast_sass_budget.py, sm_90a cross-compile, no GPU).

Pass A screens every pixel of a cell, so its instructions per pixel bound the kernel's issue time at level 0. Before the 8-pixel
items it took 207 SASS per 4-pixel item in orb_fast_cells<true> (51.8 per pixel) and 263 in orb_fast_cells<false> (65.8; that
instantiation is capped at 48 registers), at 64 and 48 registers. Both now run at 48 registers, 5 CTAs per SM, which on an H100
measured faster than the 74 registers the 8-pixel items take unbounded, though the cap adds address arithmetic to pass A. These
bounds keep a later change from silently undoing either the instruction cut or the occupancy.
"""
import os
import shutil
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools import fast_sass_budget  # noqa: E402

# CTAs of orb_fast_cells that the register file must hold per SM (both instantiations are bounded for 5)
MIN_CTAS_PER_SM = 5
# SASS per pixel of pass A, per candidate of pass B, per 32-pixel word of pass C; CTA barriers per kernel
LIMITS = {
    "tma": {"pass_a_per_px": 36.0, "pass_b_per_candidate": 105, "pass_c_per_word": 225, "bar_sync": 5},
    "plain": {"pass_a_per_px": 36.0, "pass_b_per_candidate": 105, "pass_c_per_word": 225, "bar_sync": 4},
}


@pytest.fixture(scope="module")
def budget():
    if not (shutil.which("nvcc") or os.path.exists("/usr/local/cuda/bin/nvcc")):
        pytest.skip("nvcc not found")
    return fast_sass_budget.budget()


@pytest.mark.parametrize("kernel", sorted(LIMITS))
def test_every_pass_loop_was_found(budget, kernel):
    r = budget[kernel]
    assert r["pass_a_per_item"] and r["pass_b_per_candidate"] and r["pass_c_per_word"] and r["registers"], r
    assert r["pass_a_px_per_item"] == 8   # one predicated list store per pixel of an item


@pytest.mark.parametrize("kernel", sorted(LIMITS))
def test_register_file_holds_five_ctas(budget, kernel):
    # 256-thread CTAs; the register file of an SM has 64 K registers, allocated per warp in units of 256 (8 per thread)
    per_cta = -(-budget[kernel]["registers"] // 8) * 8 * 256
    assert 65536 // per_cta >= MIN_CTAS_PER_SM, (kernel, budget[kernel]["registers"])


@pytest.mark.parametrize("kernel", sorted(LIMITS))
def test_pass_budgets(budget, kernel):
    r, lim = budget[kernel], LIMITS[kernel]
    for key, bound in lim.items():
        assert r[key] <= bound, (kernel, key, r[key], bound)
