"""The oracle against the unmodified reference's own outputs (tests/golden/reference_steps.npz, recorded from the
reference by oracle/make_golden.py)."""
import numpy as np
import pytest
import torch

from helpers import DTYPES, bits
from oracle import blend, synth, tiling
from oracle.make_golden import REF_SCATTER_CASE, REF_STEP_CASE


@pytest.fixture(scope="module")
def gold(golden_dir):
    import os
    return np.load(os.path.join(golden_dir, "reference_steps.npz"))


@pytest.mark.parametrize("method", ["md", "mod"])
@pytest.mark.parametrize("dn", list(DTYPES))
def test_step_matches_reference(gold, method, dn):
    N, C, W, H, tw, th, ov, bs = REF_STEP_CASE
    x = synth.latent(11, (N, C, H, W), DTYPES[dn])
    plan = tiling.GridPlan(W, H, tw, th, ov, bs, method == "mod")
    assert [tuple(b) for b in gold[f"{method}_{dn}_bboxes"].tolist()] == plan.bboxes
    den = lambda t, bb: synth.fake_denoise(t, bb, N)
    if method == "md":
        got = blend.multidiffusion_step(x, plan.batched_bboxes, plan.weights, den)
    else:
        got = blend.mixture_step(x, plan.batched_bboxes, plan.tile_weights, plan.rescale_factor, den)
    assert str(got.dtype) == str(gold[f"{method}_{dn}_dtype"])
    assert np.array_equal(bits(got), gold[f"{method}_{dn}"]), f"{method}/{dn}: oracle step differs from the reference's"


def test_scatter_matches_reference_cat(gold):
    N, C, W, H, tw, th, ov = REF_SCATTER_CASE
    x = synth.latent(5, (N, C, H, W), torch.float16)
    bbs = [tuple(b) for b in gold["scatter_bboxes"].tolist()]
    got = blend.scatter_tiles(x, bbs)
    assert np.array_equal(bits(got), gold["scatter"])
