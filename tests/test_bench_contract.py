"""bench.py's reference arm runs on host cores only, so its JSON line can be checked without a GPU: the keys the
driver reads, the metric / config naming shared with the GPU arm, and the oracle-only import rule of the GPU arm."""
import json
import os
import re
import subprocess
import sys

from conftest import ROOT


def test_reference_arm_prints_one_contract_line():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "2", "--warmup", "1"],
                         capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [ln for ln in out.stdout.splitlines() if ln.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["n_gpus"] == 1 and d["steps"] == 2 and d["warmup"] == 1
    assert d["metric"].startswith("megapixels/sec") and d["unit"] == "MP/s" and d["higher_is_better"] is True
    assert d["value"] > 0 and abs(d["value"] - 16.777216 / (d["ms_per_step"] * 1e-3 * 50)) / d["value"] < 1e-6   # 4096^2 image, 50 steps
    assert d["vs_baseline"] is None and d["data"].startswith("synthetic")
    assert d["e2e"] == {"value": d["value"], "unit": "MP/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    cb = d["cpu_baseline"]
    # the unmodified reference when its tree is present, else its op-for-op restatement
    from oracle import ref_shim
    assert cb["kind"] == ("reference" if ref_shim.available() else "port")
    assert cb["cores"] >= 1 and cb["value"] == d["value"] and "sample" in cb
    assert d["config"]["workload"].startswith("SD1.5 4096x4096") and (d["config"]["H"], d["config"]["W"], d["config"]["tile"]) == (512, 512, 96)


def test_gpu_arm_takes_nothing_from_the_oracle():
    """Only the cpu_baseline / reference legs may execute oracle/ (they ARE the CPU restatement being timed)."""
    src = open(os.path.join(ROOT, "bench.py")).read()
    for m in re.finditer(r"from oracle import [^\n]+", src):
        head = src[:m.start()]
        fn = re.findall(r"\ndef (\w+)\(", head)[-1]
        assert fn in ("cpu_reference_step_fn", "eager_cuda_baseline", "vae_cpu_baseline", "demofusion_cpu_baseline"), f"`{m.group(0)}` inside {fn}(): the GPU arm must not use the oracle"
    assert "import oracle" not in src
