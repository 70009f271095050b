"""Per-element comparison of GPU stage outputs with their fp64 references (tests/stage_refs.py), shared by the stage
isolation tests of the bf16 path (test_gpu_stage_isolation.py) and of the f32-class paths (test_gpu_x3_stage_isolation.py).

A Checker compares one test case stage by stage against a table of bounds, stage -> (storage ulps, c):
  stored outputs (ulps > 0):  ulps * storage_ulp(|ref|) + c * acc   per element
  f32 outputs (ulps == 0):    c * acc per element, and relative L2 <= l2_limit (default 1e-4)
It collects every failure of the case before asserting and appends one report row per stage to build/<report>, the file
truncated once per test session.

Test infrastructure only (imported by tests/)."""
import json
import math
import os
import time

import numpy as np
import pytest
import torch

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


def _pow2_floor_log2(x, shift):
    """2^(floor(log2 max(|x|, 2^-126)) + shift) of a torch tensor, on its device (the power of two built exactly)."""
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126))).long() + shift
    return ((e + 1023) << 52).view(torch.float64)


def ulp_bf16(x):
    if isinstance(x, torch.Tensor):
        return _pow2_floor_log2(x, -7)
    a = np.maximum(np.abs(x), 2.0 ** -126)
    return 2.0 ** (np.floor(np.log2(a)) - 7)


def ulp_split(x):
    """One ulp of the lo half of a split-bf16 [hi | lo] value: 2^-8 of the bf16 ulp of |x|."""
    return ulp_bf16(x) * 2.0 ** -8


def ulp_tf32(x):
    if isinstance(x, torch.Tensor):
        return _pow2_floor_log2(x, -10)
    a = np.maximum(np.abs(x), 2.0 ** -126)
    return 2.0 ** (np.floor(np.log2(a)) - 10)


_COUNTS = ("mismatches", "out_of_range", "wrong_clear", "wrong_near_tie", "live", "carry_recovered", "carry_fallbacks",
           "near_midpoint_partials")


def _larger(new, old):
    """Whether a merged maximum takes `new`: NaN beats every number and, once stored, is never replaced."""
    return not math.isnan(old) and (math.isnan(new) or new > old)


class Checker:
    """close / close_scaled / exact take numpy arrays or torch tensors; torch tensors are reduced on their own device.
    Checking the same stage again (the next image chunk of a batch checked in parts) merges into that stage's row: the
    worse element, the larger maxima, the summed counts and the relative L2 of the union."""

    def __init__(self, case, bounds, report="stage_isolation_report.jsonl", ulp=ulp_bf16, l2_limit=None):
        self.case = case
        self.bounds = bounds
        self.report_name = report
        self.ulp = ulp
        self.l2_limit = l2_limit or {}
        self._rows = {}

    @property
    def rows(self):
        return list(self._rows.values())

    @property
    def fail(self):
        out = []
        for row in self._rows.values():
            kv = {k: v for k, v in row.items() if k not in ("case", "stage", "max_ratio", "l2_limit") and k[0] != "_"}
            if "rel_l2" in row and row["rel_l2"] > row["l2_limit"]:
                out.append(f"{row['stage']}: relative L2 {row['rel_l2']:.3g} > {row['l2_limit']:g}")
            if not row["max_ratio"] <= 1.0:
                out.append(f"{row['stage']}: max |gpu-ref|/bound = {row['max_ratio']:.3g} {kv}")
        return out

    def _record(self, stage, ratio, **kv):
        ratio = float(ratio)
        row = self._rows.get(stage)
        if row is None:
            self._rows[stage] = dict(case=self.case, stage=stage, max_ratio=ratio, **kv)
            return
        # the same stage again (the next image chunk): it must be the same kind of check
        assert kv.keys() <= row.keys(), f"{stage}: checked with different kinds of check ({sorted(kv)} vs {sorted(row)})"
        worse = _larger(ratio, row["max_ratio"])
        for k, v in kv.items():
            if k in _COUNTS or k in ("_err_sq", "_ref_sq"):
                row[k] += v
            elif k in ("max_abs_err", "c_needed"):
                row[k] = v if _larger(v, row[k]) else row[k]
            elif k.startswith("worst_") and worse:
                row[k] = v
        if worse:
            row["max_ratio"] = ratio
        if "_err_sq" in row:
            row["rel_l2"] = float(np.sqrt(row["_err_sq"]) / max(np.sqrt(row["_ref_sq"]), 1e-30))

    def close(self, stage, gpu, ref, acc, key=None, mask=None):
        """Stored (ulps > 0) or f32 (ulps == 0) output against the fp64 reference, per element."""
        if isinstance(ref, torch.Tensor):
            return self._close_torch(stage, gpu, ref, acc, key, mask)
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
            en, rn = float(np.linalg.norm(g - r)), float(np.linalg.norm(r))
            kv.update(rel_l2=en / max(rn, 1e-30), l2_limit=self.l2_limit.get(key or stage, 1e-4), _err_sq=en * en,
                      _ref_sq=rn * rn)
        self._record(stage, float(ratio.max()), **kv)

    def _close_torch(self, stage, gpu, ref, acc, key, mask):
        """close() on torch tensors, reduced on ref's device: the same row as the numpy path."""
        ulps, c = self.bounds[key or stage]
        r = ref.to(torch.float64)
        g = torch.as_tensor(gpu).to(r.device, torch.float64)
        a = torch.as_tensor(acc, dtype=torch.float64, device=r.device).expand(r.shape)
        if mask is not None:
            mask = torch.as_tensor(mask, device=r.device)
            g, r, a = g[mask], r[mask], a[mask]
        if r.numel() == 0:
            return
        err = (g - r).abs()
        share = ulps * self.ulp(r) if ulps else 0.0
        bound = share + c * a if ulps else c * a + 1e-30
        ratio = err / bound
        i = int(ratio.reshape(-1).argmax())
        kv = dict(max_abs_err=float(err.max()), worst_gpu=float(g.reshape(-1)[i]), worst_ref=float(r.reshape(-1)[i]),
                  worst_acc=float(a.reshape(-1)[i]), ulps=ulps, c=c,
                  c_needed=float(((err - share).clamp_min(0.0) / a.clamp_min(1e-300)).max()))
        if not ulps:
            en, rn = float(torch.linalg.vector_norm(g - r)), float(torch.linalg.vector_norm(r))
            kv.update(rel_l2=en / max(rn, 1e-30), l2_limit=self.l2_limit.get(key or stage, 1e-4), _err_sq=en * en,
                      _ref_sq=rn * rn)
        self._record(stage, float(ratio.max()), **kv)

    def close_allow(self, stage, gpu, ref, acc, allow, mask, key=None, axes=None, origin=None, **counts):
        """A stored output whose reference leaves some of the kernel's roundings to a per-element allowance `allow`
        (stage_refs.bptt_steps_isolated): bound ulps * ulp(|ref| + allow) + allow + c * acc on the elements where `mask`
        holds (the ulp of the largest value the kernel's result may take before it is stored).
        c_needed is the part of the error neither the ulps nor the allowance cover, over acc.  Torch tensors of one shape
        (acc, allow, mask broadcast to it).  axes names the dimensions for the worst element's coordinates (worst_at), and
        origin is added to them (the first image of a chunk).  counts: extra totals for the row (_COUNTS)."""
        ulps, c = self.bounds[key or stage]
        r = ref.to(torch.float64)
        g = gpu.to(r.device, torch.float64)
        a = acc.to(r.device, torch.float64).expand(r.shape)
        al = allow.to(r.device, torch.float64).expand(r.shape)
        m = mask.to(r.device).expand(r.shape)
        if not bool(m.any()):
            return
        zero = r.new_zeros(())
        err = torch.where(m, (g - r).abs(), zero)
        share = ulps * self.ulp(r.abs() + al) + al          # the allowance may carry the stored value up a binade
        ratio = torch.where(m, err / (share + c * a + 1e-30), zero)
        ratio = torch.where(torch.isnan(ratio), float("inf"), ratio)                 # a NaN from the GPU is the worst
        i = int(ratio.reshape(-1).argmax())
        at = [int(v) for v in np.unravel_index(i, tuple(r.shape))]
        at = [v + int(o) for v, o in zip(at, origin or [0] * len(at))]
        kv = dict(max_abs_err=float(err.max()), worst_gpu=float(g.reshape(-1)[i]), worst_ref=float(r.reshape(-1)[i]),
                  worst_acc=float(a.reshape(-1)[i]), worst_allow=float(al.reshape(-1)[i]),
                  worst_at=dict(zip(axes or [f"dim{k}" for k in range(len(at))], at)), ulps=ulps, c=c,
                  c_needed=float(torch.where(m, (err - share).clamp_min(0.0) / a.clamp_min(1e-300), zero).max()),
                  **counts)
        self._record(stage, float(ratio.reshape(-1)[i]), **kv)

    def l2(self, stage, gpu, ref, key=None):
        """The relative L2 of an f32 output against its reference on its own, limit l2_limit[key or stage] (the
        per-element bounds are other stages' rows).  Torch tensors."""
        r = ref.to(torch.float64)
        g = gpu.to(r.device, torch.float64)
        en, rn = float(torch.linalg.vector_norm(g - r)), float(torch.linalg.vector_norm(r))
        self._record(stage, 0.0, rel_l2=en / max(rn, 1e-30), l2_limit=self.l2_limit.get(key or stage, 1e-4), _err_sq=en * en,
                     _ref_sq=rn * rn)

    def close_scaled(self, stage, gpu, ref, mask=None, key=None):
        """Recurrence / BPTT: bound ulps * ulp(|ref|) + c * max|ref|."""
        if isinstance(ref, torch.Tensor):
            r = ref if mask is None else ref[torch.as_tensor(mask, device=ref.device)]
            return self.close(stage, gpu, ref, float(r.abs().max()) if r.numel() else 0.0, mask=mask, key=key)
        r = np.asarray(ref, np.float64)
        self.close(stage, gpu, ref, np.abs(r[mask] if mask is not None else r).max(), mask=mask, key=key)

    def exact(self, stage, gpu, ref):
        if isinstance(gpu, torch.Tensor):
            bad = int((gpu != torch.as_tensor(ref, device=gpu.device)).sum())
        else:
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
            for row in self._rows.values():
                f.write(json.dumps(dict(run=run, **{k: v for k, v in row.items() if k[0] != "_"})) + "\n")

    def assert_ok(self):
        self.report()
        assert not self.fail, "\n".join(self.fail)
