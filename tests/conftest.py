import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def pytest_terminal_summary(terminalreporter, exitstatus, config):
    """Forward-level parity numbers (tests/util.record_parity) as a table in the log, -q or not."""
    try:
        sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
        from util import PARITY_ROWS
    except Exception:
        return
    if not PARITY_ROWS:
        return
    tr = terminalreporter
    tr.write_line("")
    tr.write_line("parity vs the fp32 reference (max / mean abs error; 'viol' = fraction outside rtol=1e-3, atol=1e-4; "
                  "stock = same op sequence through cuDNN/cuBLAS/SDPA in the same 16-bit dtype)")
    tr.write_line(f"{'case':<34}{'stage':<18}{'|ref|':>9} {'ours max':>10}{'ours mean':>11}{'viol':>8} "
                  f"{'stock max':>11}{'stock mean':>11}{'viol':>8}")
    for r in PARITY_ROWS:
        st = (f"{r['stock_max']:>11.3e}{r['stock_mean']:>11.3e}{r['stock_viol']:>8.4f}" if "stock_max" in r else "")
        tr.write_line(f"{r['case']:<34}{r['stage']:<18}{r['ref_abs_mean']:>9.4f} {r['ours_max']:>10.3e}"
                      f"{r['ours_mean']:>11.3e}{r['ours_viol']:>8.4f} {st}")
