"""Shared helpers: build the named tiny fixtures for the oracle and for the CUDA engine."""
import os
import random
import tempfile

import torch

from oracle import eagle_oracle as orc
from oracle.make_golden import FIXTURES, STOP_FIXTURES, base_fixture, fixture_models, make_prompt

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
# informational parity notes of the GPU tests (what agreed with the reference and how closely), outside the source tree
REPORT = os.path.join(tempfile.gettempdir(), "eagle_b200_parity_report.txt")
_report_started = False


def report(line: str):
    """Add one line to REPORT; the first call of a test process starts the file afresh."""
    global _report_started
    with open(REPORT, "a" if _report_started else "w") as f:
        f.write(line + "\n")
    _report_started = True


def load_golden(name):
    return torch.load(os.path.join(GOLD, name + ".pt"), weights_only=False)


def model_name(fx):
    return base_fixture(fx)


def to_cfg(d: dict) -> orc.ModelCfg:
    keys = orc.ModelCfg.__dataclass_fields__.keys()
    return orc.ModelCfg(**{k: v for k, v in d.items() if k in keys})


def build_oracle(fx):
    tcfg, tW, hcfg, hW, eagle3, dtype, tree = fixture_models(model_name(fx))
    m = orc.OracleEaModel(to_cfg(tcfg), tW, to_cfg(hcfg), hW, eagle3, **tree)
    return m, (tcfg, tW, hcfg, hW, eagle3, dtype, tree)
