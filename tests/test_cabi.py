"""The C-ABI library loads and exports every symbol include/td_b200.h declares (no GPU needed)."""
import ctypes
import os
import re

from conftest import ROOT


def _declared():
    src = open(os.path.join(ROOT, "include", "td_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(td_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_exported_and_bound():
    from multidiffusion_upscaler_for_automatic1111_b200 import _cabi
    declared = _declared()
    assert len(declared) >= 10
    raw = ctypes.CDLL(_cabi.LIB_PATH)
    for name in declared:
        assert hasattr(raw, name), f"{name} declared in td_b200.h but not exported by libtd_b200.so"
    assert sorted(_cabi.exported_symbols()) == declared, "ctypes binding and header disagree"


def test_abi_version_and_error_string():
    from multidiffusion_upscaler_for_automatic1111_b200 import _cabi
    assert _cabi.lib.td_abi_version() == _cabi.ABI_VERSION
    st = _cabi.lib.td_split_bboxes(64, 64, 16, 16, 16, None, 0, None, None)  # overlap == tile: invalid
    assert st == _cabi.TD_ERR_INVALID_ARG
    assert b"overlap" in _cabi.lib.td_last_error()


def test_grid_struct_layout_matches_header():
    from multidiffusion_upscaler_for_automatic1111_b200 import _cabi
    assert ctypes.sizeof(_cabi.TdGrid) == 4 * (11 + 2 * _cabi.TD_MAX_GRID_DIM)
    assert _cabi.TdGrid.wrap.offset == 4 * 10 and _cabi.TdGrid.ys.offset == 4 * 11


def test_region_struct_layout_matches_header():
    """struct td_region: five int32 geometry / mode fields, the output's dtype in what used to be padding, two pointers."""
    from multidiffusion_upscaler_for_automatic1111_b200 import _cabi
    assert ctypes.sizeof(_cabi.TdRegion) == 40
    assert [(n, getattr(_cabi.TdRegion, n).offset) for n, _ in _cabi.TdRegion._fields_] == \
        [("x", 0), ("y", 4), ("w", 8), ("h", 12), ("mode", 16), ("dtype", 20), ("out", 24), ("aux", 32)]
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "td_b200.h")).read(), flags=re.S)
    body = re.search(r"typedef struct td_region \{(.*?)\} td_region;", src, flags=re.S).group(1)
    declared = [n for decl in body.split(";") if decl.strip() for n in re.findall(r"\*?\s*(\w+)\s*(?:,|$)", decl.strip())]
    assert declared == [n for n, _ in _cabi.TdRegion._fields_], f"header fields {declared}"


def test_missing_library_fails_loudly(tmp_path, monkeypatch):
    """No silent fallback: a missing .so is an ImportError naming the build command."""
    import importlib

    from multidiffusion_upscaler_for_automatic1111_b200 import _cabi
    monkeypatch.setattr(_cabi, "LIB_PATH", str(tmp_path / "nope.so"))
    try:
        _cabi._load()
    except ImportError as e:
        assert "no CPU" in str(e) or "fallback" in str(e)
    else:
        raise AssertionError("loading a missing library must raise")
    importlib.reload  # keep linters quiet
