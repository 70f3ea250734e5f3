"""CPU checks of the bench.py contract that do not need a GPU: the reference arm (the oracle timed on the host cores) prints one
well-formed JSON line, non-zero ranks of a torchrun launch stay silent and exit 0, and the product arm refuses to run without
a CUDA device instead of falling back to anything."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(args, env=None, timeout=600):
    e = dict(os.environ)
    e.update(env or {})
    return subprocess.run([sys.executable, os.path.join(ROOT, "bench.py")] + args, capture_output=True, text=True, env=e,
                          timeout=timeout, cwd=ROOT)


def test_reference_arm_prints_contract_line():
    r = _run(["--impl", "reference", "--size", "64", "--steps", "4", "--warmup", "0"])
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == "512x512 images/sec" and d["unit"] == "images/s"
    assert d["value"] > 0 and d["ms_per_step"] > 0 and d["higher_is_better"] is True and d["n_gpus"] == 1
    assert d["steps"] == 4 and d["warmup"] == 0                       # --steps / --warmup are timed as given, never clamped
    assert d["e2e"] == {"value": d["value"], "unit": "images/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    cb = d["cpu_baseline"]
    assert cb["kind"] == "port" and cb["cores"] >= 1 and cb["value"] == d["value"] and "sample" in cb
    assert "workload" in d["config"] and "model" not in d["config"]


def test_steps_that_cannot_be_honoured_are_rejected():
    for args in (["--steps", "0"], ["--warmup", "-1"]):
        r = _run(["--impl", "reference", "--size", "64"] + args)
        assert r.returncode != 0 and "{" not in r.stdout and "--steps must be" in r.stderr


def test_reference_arm_other_ranks_are_silent():
    r = _run(["--impl", "reference", "--gpus", "2", "--steps", "1", "--warmup", "1"], env={"RANK": "1", "WORLD_SIZE": "2",
                                                                                            "LOCAL_RANK": "1"})
    assert r.returncode == 0 and r.stdout.strip() == ""


def test_product_arm_needs_a_gpu():
    import torch
    if torch.cuda.is_available():
        return
    r = _run(["--steps", "1", "--warmup", "1"], timeout=300)
    assert r.returncode != 0 and "{" not in r.stdout          # no number is printed, nothing falls back to the CPU
