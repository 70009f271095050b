"""Per-element comparison of GPU stage outputs with their fp64 references (tests/stage_refs.py), shared by the stage
isolation tests of the bf16 path (test_gpu_stage_isolation.py) and of the f32-class paths (test_gpu_x3_stage_isolation.py).

A Checker compares one test case stage by stage against a table of bounds, stage -> (storage ulps, c):
  stored outputs (ulps > 0):  ulps * storage_ulp(|ref|) + c * acc   per element
  f32 outputs (ulps == 0):    c * acc per element, and relative L2 <= l2_limit (default 1e-4)
It collects every failure of the case before asserting and appends one report row per stage to build/<report>, the file
truncated once per test session.

Test infrastructure only (imported by tests/)."""
import json
import os
import time

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_REPORT_RUN = {}            # report file -> start time of this session's report (each file is truncated once per session)

# shapes of the stage isolation tests: every mg2/mg3/mg4 value, two 128-row tiles, lengths 0, 1, T and in between
SHAPES = [
    pytest.param(2, 256, [256, 201], id="N2_W256"),
    pytest.param(3, 160, [160, 8, 97], id="N3_W160"),
    pytest.param(5, 80, [80, 4, 8, 57, 33], id="N5_W80"),
    pytest.param(3, 100, [100, 4, 61], id="N3_W100"),
    pytest.param(130, 40, "cycle", id="N130_W40"),
    pytest.param(5, 24, [24, 4, 8, 12, 20], id="N5_W24"),
]


def widths_of(N, W, widths):
    if widths == "cycle":                                  # lengths 0, 1, T and in between, over two 128-row tiles
        return [[W, 4, 8, 12, 20, 28, 36][i % 7] for i in range(N)]
    return widths


def ulp_bf16(x):
    a = np.maximum(np.abs(x), 2.0 ** -126)
    return 2.0 ** (np.floor(np.log2(a)) - 7)


def ulp_split(x):
    """One ulp of the lo half of a split-bf16 [hi | lo] value: 2^-8 of the bf16 ulp of |x|."""
    return ulp_bf16(x) * 2.0 ** -8


def ulp_tf32(x):
    a = np.maximum(np.abs(x), 2.0 ** -126)
    return 2.0 ** (np.floor(np.log2(a)) - 10)


class Checker:
    def __init__(self, case, bounds, report="stage_isolation_report.jsonl", ulp=ulp_bf16, l2_limit=None):
        self.case = case
        self.bounds = bounds
        self.report_name = report
        self.ulp = ulp
        self.l2_limit = l2_limit or {}
        self.fail = []
        self.rows = []

    def _record(self, stage, ratio, **kv):
        self.rows.append(dict(case=self.case, stage=stage, max_ratio=float(ratio), **kv))
        if not ratio <= 1.0:
            self.fail.append(f"{stage}: max |gpu-ref|/bound = {ratio:.3g} {kv}")

    def close(self, stage, gpu, ref, acc, key=None, mask=None):
        """Stored (ulps > 0) or f32 (ulps == 0) output against the fp64 reference, per element."""
        ulps, c = self.bounds[key or stage]
        g, r = np.asarray(gpu, np.float64), np.asarray(ref, np.float64)
        a = np.broadcast_to(np.asarray(acc, np.float64), r.shape)
        if mask is not None:
            g, r, a = g[mask], r[mask], a[mask]
        if r.size == 0:
            return
        err = np.abs(g - r)
        bound = ulps * self.ulp(r) + c * a if ulps else c * a + 1e-30
        ratio = err / bound
        i = int(np.argmax(ratio))
        # c_needed: the smallest c that would hold every element (the part of the error the storage ulps do not cover)
        c_needed = float((np.maximum(err - (ulps * self.ulp(r) if ulps else 0.0), 0.0) / np.maximum(a, 1e-300)).max())
        kv = dict(max_abs_err=float(err.max()), worst_gpu=float(g.flat[i]), worst_ref=float(r.flat[i]),
                  worst_acc=float(a.flat[i]), ulps=ulps, c=c, c_needed=c_needed)
        if not ulps:
            l2 = float(np.linalg.norm(g - r) / max(np.linalg.norm(r), 1e-30))
            kv["rel_l2"] = l2
            lim = self.l2_limit.get(key or stage, 1e-4)
            if l2 > lim:
                self.fail.append(f"{stage}: relative L2 {l2:.3g} > {lim:g}")
        self._record(stage, float(ratio.max()), **kv)

    def close_scaled(self, stage, gpu, ref, mask=None, key=None):
        """Recurrence / BPTT: bound ulps * ulp(|ref|) + c * max|ref|."""
        r = np.asarray(ref, np.float64)
        self.close(stage, gpu, ref, np.abs(r[mask] if mask is not None else r).max(), mask=mask, key=key)

    def exact(self, stage, gpu, ref):
        g, r = np.asarray(gpu), np.asarray(ref)
        bad = int((g != r).sum())
        self._record(stage, 0.0 if bad == 0 else float("inf"), mismatches=bad)

    def report(self):
        """Rows of this test session only: the first report of a session truncates the file, every row carries the
        session's start time."""
        os.makedirs(os.path.join(ROOT, "build"), exist_ok=True)
        mode = "a" if self.report_name in _REPORT_RUN else "w"
        run = _REPORT_RUN.setdefault(self.report_name, time.strftime("%Y-%m-%dT%H:%M:%S"))
        with open(os.path.join(ROOT, "build", self.report_name), mode) as f:
            for row in self.rows:
                f.write(json.dumps(dict(run=run, **row)) + "\n")

    def assert_ok(self):
        self.report()
        assert not self.fail, "\n".join(self.fail)
