"""CPU: LRSchedule vs the trace of the reference's own class committed in tests/golden/lr_schedule.json (written by
oracle/make_golden_host.py, never by a test)."""
import json
import os

from latex_ocr_b200.lr_schedule import LRSchedule
from oracle import make_golden_host as mgh

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lr_schedule.json")


def _close(got, want):
    for (lr, stop), (wlr, wstop) in zip(got, want):
        assert abs(lr - wlr) <= 1e-15 + 1e-12 * abs(wlr) and stop == bool(wstop), (got, want)


def test_lr_schedule_matches_reference():
    for kw, want in zip(mgh.LR_CASES, json.load(open(GOLD))):
        _close(mgh.lr_trace(LRSchedule, kw), want)
