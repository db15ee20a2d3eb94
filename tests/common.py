"""Shared helpers for tests: golden loading + case reconstruction (inputs are re-generated from seeds)."""
import json
import os

import torch

from mvsformerplusplus_b200 import synth
from mvsformerplusplus_b200.config import default_args
from mvsformerplusplus_b200.params import build_hotpath_params
from oracle import fixture

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TMP = [5.0, 5.0, 5.0, 1.0]


def load_golden(name):
    """-> ({name: CPU tensor}, meta) of tests/golden/<name>.npz"""
    arrays, meta = fixture.load(os.path.join(GOLDEN, name + ".npz"))
    return {k: torch.from_numpy(v) for k, v in arrays.items()}, meta


def build_case(meta, args=None):
    """Re-creates exactly the inputs oracle/gen_golden.py used (same seeds, same generators)."""
    args = args or default_args()
    feats = synth.make_features(meta["V"], meta["H"], meta["W"], seed=meta["fseed"])
    proj = synth.make_proj_matrices(meta["V"], meta["H"], meta["W"], theta_step=0.12)
    dv = synth.make_depth_values(meta["numdepth"], 425.0, 2.65 * 192 / meta["numdepth"])
    torch.manual_seed(0)
    params = build_hotpath_params(args).eval()
    sd = synth.randomize_state_dict(params, seed=meta["wseed"])
    return args, params, sd, feats, proj, dv


def max_abs(a, b):
    return float((a.double() - b.double()).abs().max())


def rel_linf(a, b):
    return float(((a.double() - b.double()).abs() / b.double().abs().clamp_min(1e-12)).max())


# ---- error reports of the GPU test modules, written as the tests run: $MVSF_TEST_REPORT_DIR, else test_reports/ in the
#      repository (git-ignored)
REPORT = {}
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REPORT_DIR = os.environ.get("MVSF_TEST_REPORT_DIR") or os.path.join(ROOT, "test_reports")


def rec(name, **kw):
    REPORT[name] = {k: (float(v) if isinstance(v, (int, float)) else v) for k, v in kw.items()}
    os.makedirs(REPORT_DIR, exist_ok=True)
    with open(os.path.join(REPORT_DIR, "parity_report.json"), "w") as f:
        json.dump(REPORT, f, indent=1, sort_keys=True)
