"""ControlNet / StableSR tile caches (SURVEY.md section 8(f)-2): the per-batch hint tiles our delegate caches and
hands to the extension objects must equal the reference's, for k-diffusion and DDIM samplers, grid and custom bboxes.

CPU: our delegate under the stub host (oracle/ref_shim.py), with the scatter kernel swapped for the oracle's scatter
(the kernel itself is pinned by tests/test_gpu_diffusion.py), against the UNMODIFIED reference's caches in the same
sequence of calls, recorded by `reference_records` (oracle/make_golden.py -> tests/golden/host_records.npz).  GPU: the
same caches through td_scatter_tiles on the x8-scaled tile plan, against plain slicing.
"""
import types

import pytest
import torch

from helpers import digest, host_record
from oracle import blend, ref_shim

W, H = 64, 48
ROWS = [(True, 0.1, 0.2, 0.5, 0.4, "a cat", "", "Background", 0.2, -1),
        (True, 0.4, 0.3, 0.45, 0.6, "a dog", "ugly", "Foreground", 0.3, 5)]


def _p():
    return types.SimpleNamespace(width=W * 8, height=H * 8, sampler_name="Euler a", disable_extra_networks=True,
                                 batch_size=1, steps=20, styles=None, all_prompts=["a photo"], all_negative_prompts=["blurry"])


def _hints(device="cpu"):
    a = (torch.arange(1 * 3 * H * 8 * W * 8, dtype=torch.float32, device=device).view(1, 3, H * 8, W * 8) % 1021) / 1021.0
    b = (torch.arange(3 * H * 8 * W * 8, dtype=torch.float32, device=device).view(3, H * 8, W * 8) % 509) / 509.0   # 3-d: unsqueezed in place
    return [a, b]


def _controlnet_script(device="cpu"):
    params = [types.SimpleNamespace(hint_cond=t) for t in _hints(device)]
    return types.SimpleNamespace(latest_network=types.SimpleNamespace(control_params=params))


def _oracle_scatter(monkeypatch):
    from multidiffusion_upscaler_for_automatic1111_b200 import engine

    def scatter_tiles(g, x, out=None, tile_begin=0, tile_end=None, flags=0):
        bbs = [tuple(int(v) for v in r) for r in engine.grid_bboxes_xywh(g)]
        return blend.scatter_tiles(x, bbs[tile_begin:tile_end])
    monkeypatch.setattr(engine, "scatter_tiles", scatter_tiles)


def _delegate(cls, sampler, settings, with_regions):
    d = cls(_p(), sampler)
    d.init_grid_bbox(16, 16, 8, 4)
    if with_regions:
        d.init_custom_bbox(settings, True, False)
    return d


def _settings(ref):
    if ref is None:
        from multidiffusion_upscaler_for_automatic1111_b200 import MultiDiffusion
        return MultiDiffusion, {i: r for i, r in enumerate(ROWS)}
    return ref.multidiffusion.MultiDiffusion, {i: ref.utils.BBoxSettings(*r) for i, r in enumerate(ROWS)}


CONTROLNET_CASES = [(kdiff, with_regions, tensor_cpu) for tensor_cpu in (False, True) for with_regions in (False, True) for kdiff in (True, False)]


def _controlnet_trace(kdiff, with_regions, tensor_cpu, ref=None):
    """Digests of every hint tensor our delegate (or the reference's, `ref` given) caches and hands to the ControlNet
    script, in call order."""
    from multidiffusion_upscaler_for_automatic1111_b200 import host
    stubs = ref_shim.host_stubs()
    host._a1111_cache.clear()
    if kdiff:
        sampler = ref_shim.make_kdiff_sampler(lambda x, s, cond=None: x)
    else:
        class _S(stubs.CompVisSampler):
            pass
        sampler = _S()
        sampler.model_wrap_cfg = types.SimpleNamespace(inner_model=types.SimpleNamespace(forward=None), image_cfg_scale=None, step=0)
    cls, settings = _settings(ref)
    d = _delegate(cls, sampler, settings, with_regions)
    assert d.is_kdiff == kdiff
    cs = _controlnet_script()
    d.init_controlnet(cs, tensor_cpu)
    d.init_done()
    if getattr(d, "pbar", None) is not None:
        d.pbar.disable = True
    trace = [d.num_batches, [len(bb) for bb in d.batched_bboxes]]
    assert len(d.control_tensor_batch) == 2
    trace.append(("batch", [list(pr) for pr in d.control_tensor_batch]))
    if with_regions:
        trace.append(("custom", [list(pr) for pr in d.control_tensor_custom]))
    for batch_id in (0, d.num_batches - 1):
        n_tiles = len(d.batched_bboxes[batch_id])
        for is_denoise in (False, True):
            d.switch_controlnet_tensors(batch_id, 2, n_tiles, is_denoise=is_denoise)
            trace.append(("switch", batch_id, is_denoise, [q.hint_cond for q in cs.latest_network.control_params]))
    if with_regions:
        d.set_custom_controlnet_tensors(1, 3)
        trace.append(("set_custom", [q.hint_cond for q in cs.latest_network.control_params]))
    d.reset_controlnet_tensors()
    assert all(q.hint_cond.shape == (1, 3, H * 8, W * 8) for q in cs.latest_network.control_params)
    trace.append(("reset", [q.hint_cond for q in cs.latest_network.control_params]))
    host._a1111_cache.clear()
    return [digest(t) for t in trace]


def _stablesr_trace(ref=None):
    from multidiffusion_upscaler_for_automatic1111_b200 import host
    ref_shim.host_stubs()
    host._a1111_cache.clear()
    latent = torch.arange(2 * 4 * H * W, dtype=torch.float32).view(2, 4, H, W)
    cls, settings = _settings(ref)
    d = _delegate(cls, ref_shim.make_kdiff_sampler(lambda x, s, cond=None: x), settings, True)
    model = types.SimpleNamespace(set_image_hooks={}, latent_image=None)
    d.init_stablesr(types.SimpleNamespace(stablesr_model=model))
    d.init_done()
    if getattr(d, "pbar", None) is not None:
        d.pbar.disable = True
    model.set_image_hooks["TiledDiffusion"](latent)
    assert d.enable_stablesr
    trace = [d.num_batches, len(d.stablesr_tensor_batch)]
    for b in range(d.num_batches):
        d.switch_stablesr_tensors(b)
        trace.append(model.latent_image)
    d.set_custom_stablesr_tensors(1)
    trace.append(model.latent_image)
    d.reset_stablesr_tensors()
    assert model.latent_image is latent
    host._a1111_cache.clear()
    return [digest(t) for t in trace]


def _cn_key(kdiff, with_regions, tensor_cpu):
    return f"controlnet_{'kdiff' if kdiff else 'ddim'}_{'regions' if with_regions else 'grid'}_{'cpu' if tensor_cpu else 'dev'}"


def reference_records(ref):
    """The reference's side of every comparison below (run by oracle/make_golden.py)."""
    out = {_cn_key(*c): " ".join(_controlnet_trace(*c, ref=ref)) for c in CONTROLNET_CASES}
    out["stablesr"] = " ".join(_stablesr_trace(ref))
    return out


def _same_trace(got, want):
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"trace entry {i} differs from the reference's"


@pytest.mark.parametrize("kdiff", [True, False], ids=["kdiff", "ddim"])
@pytest.mark.parametrize("with_regions", [False, True], ids=["grid", "grid+regions"])
@pytest.mark.parametrize("tensor_cpu", [False, True], ids=["dev", "cpu_cache"])
def test_controlnet_tile_caches_like_the_reference(monkeypatch, golden_dir, kdiff, with_regions, tensor_cpu):
    _oracle_scatter(monkeypatch)
    _same_trace(_controlnet_trace(kdiff, with_regions, tensor_cpu), host_record(golden_dir, _cn_key(kdiff, with_regions, tensor_cpu)).split())


def test_stablesr_tile_caches_like_the_reference(monkeypatch, golden_dir):
    _oracle_scatter(monkeypatch)
    _same_trace(_stablesr_trace(), host_record(golden_dir, "stablesr").split())


def test_scaled_grid_is_the_tile_plan_times_opt_f():
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    g = engine.make_grid(W, H, 16, 16, 8, 4)
    s = engine.scaled_grid(g, 8)
    assert (s.H, s.W, s.tile_h, s.tile_w, s.rows, s.cols, s.num_tiles, s.tile_bs) == (H * 8, W * 8, 128, 128, g.rows, g.cols, g.num_tiles, g.tile_bs)
    assert (engine.grid_bboxes_xywh(s) == engine.grid_bboxes_xywh(g) * 8).all()
