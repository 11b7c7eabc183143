"""Region prompt control, conditioning side: `kdiff_custom_forward` / `ddim_custom_forward` must hand the UNet exactly
the rows, sigmas and cond tensors the reference hands it, for every way the k-diffusion CFG wrapper slices a batch.

Our delegate runs under the stub host of oracle/ref_shim.py (with its deterministic stand-in for the WebUI prompt
parser); its UNet calls and outputs are compared with those of the UNMODIFIED reference in the same scenarios, recorded
by `reference_records` (oracle/make_golden.py -> tests/golden/host_records.npz).
"""
import itertools
import types

import pytest
import torch

from helpers import digest, host_record
from oracle import ref_shim

W, H = 64, 48
ROWS = [(True, 0.1, 0.2, 0.5, 0.4, "a cat", "", "Background", 0.2, -1),
        (True, 0.4, 0.3, 0.45, 0.6, "a very long region prompt that spills into a second chunk of tokens", "ugly", "Foreground", 0.3, 5)]
SHORT, LONG = "a photo", "a photo of something described with so many words that the encoder needs two chunks"


@pytest.fixture()
def stubs():
    from multidiffusion_upscaler_for_automatic1111_b200 import host
    st = ref_shim.host_stubs()
    host._a1111_cache.clear()          # pick up the stub `modules.*` the shim just installed
    keep = st.shared.batch_cond_uncond
    yield st
    st.shared.batch_cond_uncond = keep
    host._a1111_cache.clear()


def _p(prompt, neg, batch_size):
    return types.SimpleNamespace(width=W * 8, height=H * 8, sampler_name="Euler a", disable_extra_networks=True,
                                 batch_size=batch_size, steps=20, styles=None,
                                 all_prompts=[f"{prompt} {i}" for i in range(batch_size)],
                                 all_negative_prompts=[f"{neg} {i}" for i in range(batch_size)])


def _delegate(prompt, neg, batch_size, edit, ref=None):
    """Our delegate, or the reference's (`ref` given), with the regions of ROWS; on CPU."""
    if ref is None:
        from multidiffusion_upscaler_for_automatic1111_b200 import MultiDiffusion as cls
        settings = {i: r for i, r in enumerate(ROWS)}
    else:
        cls, settings = ref.multidiffusion.MultiDiffusion, {i: ref.utils.BBoxSettings(*r) for i, r in enumerate(ROWS)}
    d = cls(_p(prompt, neg, batch_size), ref_shim.make_kdiff_sampler(lambda x, s, cond=None: x))
    d.init_grid_bbox(16, 16, 8, 4)
    d.init_custom_bbox(settings, True, False)
    d.init_done()
    if getattr(d, "pbar", None) is not None:
        d.pbar.disable = True
    d.is_edit_model = edit
    return d


class _Recorder:
    def __init__(self):
        self.calls = []

    def __call__(self, x, sigma, cond=None):
        tc = cond["c_crossattn"][0]
        ic = cond["c_concat"][0]
        self.calls.append((x.clone(), sigma.clone(), tc.clone(), ic.clone()))
        return x * 2 + tc.mean() + sigma.view(-1, 1, 1, 1)


def _drive(d, chunks, steps=(0, 1)):
    """Feed every region the virtual batch in `chunks` (row counts), for two sampler steps."""
    rec = _Recorder()
    outs = []
    rows = sum(chunks)
    for step in steps:
        d.sampler.model_wrap_cfg.step = step
        for bbox_id, bbox in enumerate(d.custom_bboxes):
            x_full = torch.arange(rows * 4 * bbox.h * bbox.w, dtype=torch.float32).view(rows, 4, bbox.h, bbox.w) / 1000.0 + step
            sigma = torch.arange(rows, dtype=torch.float32) + 1
            cond = {"c_crossattn": [torch.zeros(rows, 77, 8)], "c_concat": [torch.full((rows, 5, 1, 1), 0.5)]}
            lo = 0
            for n in chunks:
                outs.append(d.kdiff_custom_forward(x_full[lo:lo + n], sigma[lo:lo + n], cond, bbox_id, bbox, rec).clone())
                lo += n
    return rec.calls, outs


SCENARIOS = []
for batch_size, (prompt, neg), edit, bcu in itertools.product([1, 2], [(SHORT, SHORT), (LONG, SHORT)], [False, True], [True, False]):
    rows = batch_size * (3 if edit else 2)
    splits = {(rows,), tuple([1] * rows), (batch_size,) * (rows // batch_size)}
    if rows >= 3:
        splits.add((rows - 1, 1))
        splits.add((1, rows - 1))
    for chunks in sorted(splits):
        if bcu and len(chunks) > 1:
            continue                      # with batch_cond_uncond the wrapper always sends the whole batch at once
        SCENARIOS.append((batch_size, prompt, neg, edit, bcu, chunks))


SCENARIO_IDS = [f"bs{s[0]}_{'long' if s[1] is LONG else 'short'}_{'edit' if s[3] else 'std'}_{'bcu' if s[4] else 'seq'}_{'-'.join(map(str, s[5]))}"
                for s in SCENARIOS]
DDIM_PROMPTS = [(SHORT, SHORT), (LONG, SHORT), (SHORT, LONG)]


def _kdiff_record(sc, shared, ref=None):
    """(UNet calls, outputs) digests of one scenario, or "raises <Exception>" when the delegate cannot serve it."""
    batch_size, prompt, neg, edit, bcu, chunks = sc
    shared.batch_cond_uncond = bcu
    d = _delegate(prompt, neg, batch_size, edit, ref)
    try:
        calls, outs = _drive(d, chunks)
    except Exception as e:
        return f"raises {type(e).__name__}"
    return f"{digest(calls)} {digest(outs)}"


def _ddim_record(prompt, neg, ref=None):
    d = _delegate(prompt, neg, 1, False, ref)
    d.sampler.model_wrap_cfg.step = 3
    calls = []

    def fwd(x, cond, ts, unconditional_conditioning=None):
        calls.append((x.clone(), ts.clone(), cond["c_crossattn"][0].clone(), unconditional_conditioning["c_crossattn"][0].clone(),
                      cond["c_concat"][0].clone()))
        return x + 1
    outs = []
    for bbox in d.custom_bboxes:
        x = torch.ones(1, 4, bbox.h, bbox.w)
        cond_in = {"c_crossattn": [torch.zeros(1, 77, 8)], "c_concat": [torch.arange(5 * H * W, dtype=torch.float32).view(1, 5, H, W)]}
        outs.append(d.ddim_custom_forward(x, cond_in, bbox, torch.tensor([7]), fwd))
    return f"{digest(calls)} {digest(outs)}"


def reference_records(ref):
    """The reference's side of every comparison below (run by oracle/make_golden.py)."""
    keep = ref.shared.batch_cond_uncond
    out = {f"region_cond_kdiff_{i}": _kdiff_record(sc, ref.shared, ref) for i, sc in zip(SCENARIO_IDS, SCENARIOS)}
    ref.shared.batch_cond_uncond = keep
    out.update({f"region_cond_ddim_{k}": _ddim_record(prompt, neg, ref) for k, (prompt, neg) in enumerate(DDIM_PROMPTS)})
    return out


@pytest.mark.parametrize("sc", SCENARIOS, ids=SCENARIO_IDS)
def test_kdiff_custom_forward_feeds_the_unet_like_the_reference(stubs, golden_dir, sc):
    want = host_record(golden_dir, f"region_cond_kdiff_{SCENARIO_IDS[SCENARIOS.index(sc)]}")
    if want.startswith("raises"):    # slicings the reference itself cannot serve: nothing to compare
        pytest.skip(f"reference {want} here")
    assert _kdiff_record(sc, stubs.shared) == want


@pytest.mark.parametrize("prompt,neg", DDIM_PROMPTS)
def test_ddim_custom_forward_like_the_reference(stubs, golden_dir, prompt, neg):
    assert _ddim_record(prompt, neg) == host_record(golden_dir, f"region_cond_ddim_{DDIM_PROMPTS.index((prompt, neg))}")
