"""Differential fuzz of the oracle against the unmodified reference, replayed from what the reference computed
(tests/golden/diff_fuzz_reference.json, tests/golden/diff_fuzz_loops.pt; `python -m oracle.diff_fuzz --record` regenerates
them where the reference is importable).  Complements the other fixtures: seeded random inputs over many seeds and shapes,
values and autograd gradients of every fake-quant function plus the RTN / optimized-RTN routes must agree bit for bit."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_oracle_equals_live_reference_on_random_inputs():
    p = subprocess.run([sys.executable, "-m", "oracle.diff_fuzz", "--seeds", "6"], cwd=ROOT, capture_output=True, text=True,
                       timeout=900)
    line = [l for l in p.stdout.splitlines() if l.startswith("{")]
    assert line, p.stderr[-2000:]
    res = json.loads(line[-1])
    assert res["cases"] >= 130
    assert res["failures"] == [], res["failures"][:10]


def test_oracle_replays_live_reference_runs_with_non_default_loop_options():
    """enable_minmax_tuning=False, not_use_best_mse=True, explicit lr / minmax_lr, batch size 2, gradient_accumulate_steps=2:
    runs of the reference's AutoRound on the tiny Llama, and every block's losses and final weights are reproduced bit for
    bit by the oracle loop."""
    p = subprocess.run([sys.executable, "-m", "oracle.diff_fuzz", "--loops"], cwd=ROOT, capture_output=True, text=True, timeout=1200)
    line = [l for l in p.stdout.splitlines() if l.startswith("{")]
    assert line, p.stderr[-2000:]
    res = json.loads(line[-1])
    assert res["cases"] == 10 and res["failures"] == [], res
