"""The measurement scripts under tools/ on the host: each imports without running anything, they all time GPU work and
read the card through tools/gpu_timing.py alone, and that module refuses to time without a CUDA device."""
import importlib
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOLS = os.path.join(ROOT, "tools")
sys.path.insert(0, ROOT)
sys.path.insert(0, TOOLS)

SCRIPTS = ["time_attention", "time_bnn_mcmc", "time_conv_encoder", "time_gp_fit", "time_gp_mcmc", "time_omniglot_prior",
           "time_regression_baselines", "time_stroke_prior", "time_tabular", "step_breakdown", "sweep_wgrad_splits"]


@pytest.mark.parametrize("name", SCRIPTS)
def test_script_imports_without_running(name, capsys):
    mod = importlib.import_module(name)
    assert callable(mod.main)
    assert capsys.readouterr().out == ""


def test_card_without_cuda_names_the_tool(monkeypatch):
    import gpu_timing
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(SystemExit, match="some_tool"):
        gpu_timing.card("some_tool")


def test_only_gpu_timing_times_gpu_work_or_reads_the_card():
    found = []
    for d, dirs, files in os.walk(TOOLS):
        dirs[:] = [x for x in dirs if x != "__pycache__"]
        for f in files:
            path = os.path.join(d, f)
            if path == os.path.join(TOOLS, "gpu_timing.py"):
                continue
            with open(path, "rb") as fh:
                text = fh.read()
            found += [(os.path.relpath(path, ROOT), s) for s in ("nvidia-smi", "Event(enable_timing", "ProfilerActivity")
                      if s.encode() in text]
    assert found == []
