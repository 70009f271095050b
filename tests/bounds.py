"""Guarded buffers: where an entry point writes and what it reads, checked byte for byte.

Every caller-owned buffer is one allocation [front guard | body | back guard].  The body has exactly the size the header or the
size query gives and starts at the alignment the entry point requires; each guard is at least GUARD bytes.

  kind "out"    output or workspace: the body is filled with 0xFF before each call, the guards hold a position-dependent byte
                pattern, so a write of any value into them is seen.
  kind "state"  read and written (bound parameters, solver slots, moving statistics): the body is restored before each call,
                the guards hold the pattern, then 0xFF in the last run.
  kind "in"     input: the body is its data and ends at the back guard, which starts right after the last element.  The guards
                are zero-filled in two runs and 0xFF-filled in a third (NaN for floats, -1 for ints).

run_case makes the three runs.  After each, every guard must hold what it was armed with.  Then the rule of
test_gpu_training_run._bit_identity: what the two zero runs reproduce bit for bit must be identical in the 0xFF run (a read
past an input that reaches an output changes it), and float outputs that two runs do not reproduce must be finite.
Nothing here needs a GPU: on device "cpu" the same checks guard host buffers."""
import numpy as np
import torch

GUARD = 1 << 20
_DT = {np.dtype(np.float32): torch.float32, np.dtype(np.int32): torch.int32, np.dtype(np.int64): torch.int64,
       np.dtype(np.uint8): torch.uint8, np.dtype(np.float64): torch.float64}


def pattern(n, seed=0, device="cpu"):
    """The guard pattern: byte i is ((i + seed) * 2654435761) mod 251, so no two nearby bytes repeat a run."""
    i = torch.arange(int(n), dtype=torch.int64, device=device).add_(int(seed))
    return i.mul_(2654435761).remainder_(251).to(torch.uint8)


class Guarded:
    """One buffer of `nbytes` bytes, at `align` (absolute address), between two guards of at least `guard` bytes.
    `offset` places the body that many bytes past an aligned address (the misalignment cases)."""

    def __init__(self, name, nbytes, kind="out", align=16, guard=GUARD, device="cuda", pinned=False, dtype=torch.uint8,
                 shape=None, offset=0, compare=True, poison=0xFF):
        assert kind in ("out", "state", "in")
        self.name, self.kind, self.dtype, self.compare, self.poison = name, kind, dtype, compare, poison
        self.nbytes = int(nbytes)
        self.shape = tuple(shape) if shape is not None else None
        self.raw = torch.empty(guard + align + offset + self.nbytes + guard, dtype=torch.uint8, device=device,
                               pin_memory=pinned)
        base = self.raw.data_ptr()
        self.off = (base + guard + align - 1) // align * align - base + offset
        self.body = self.raw[self.off:self.off + self.nbytes]
        self.front, self.back = self.raw[:self.off], self.raw[self.off + self.nbytes:]
        self._pat_front = pattern(self.off, seed=len(name), device=device)
        self._pat_back = pattern(self.back.numel(), seed=len(name) + self.off + self.nbytes, device=device)
        self.saved = None
        self.arm("pattern" if kind != "in" else 0)

    @property
    def ptr(self):
        return self.raw.data_ptr() + self.off

    def view(self):
        v = self.body.view(self.dtype)
        return v.view(self.shape) if self.shape is not None else v

    def set(self, array):
        """Write the body from a host array or tensor of exactly nbytes; a state buffer keeps it to restore before each run."""
        t = torch.as_tensor(np.ascontiguousarray(array)) if not torch.is_tensor(array) else array.contiguous()
        assert t.numel() * t.element_size() == self.nbytes, (self.name, t.numel() * t.element_size(), self.nbytes)
        if self.nbytes:
            self.body.copy_(t.reshape(-1).view(torch.uint8))
        if self.kind == "state":
            self.saved = self.body.clone()
        return self

    def arm(self, fill):
        """Fill both guards with the pattern ("pattern") or a byte, or the back guard with the leading bytes of a uint8 tensor
        (the front one with 0xFF), and remember it."""
        self.armed = fill
        if torch.is_tensor(fill):
            self.front.fill_(0xFF)
            self.back.copy_(fill[:self.back.numel()])
        elif fill == "pattern":
            self.front.copy_(self._pat_front)
            self.back.copy_(self._pat_back)
        else:
            self.front.fill_(fill)
            self.back.fill_(fill)

    def prepare(self, run):
        """Before run 0, 1, 2: outputs poisoned, state restored, input guards 0, 0, then 0xFF (or the input's `poison`)."""
        if self.kind == "out":
            self.body.fill_(0xFF)
        elif self.kind == "state":
            self.body.copy_(self.saved)
            self.arm("pattern" if run < 2 else 0xFF)
        else:
            self.arm(0 if run < 2 else self.poison)

    def problems(self):
        """'' when both guards hold what they were armed with, else the buffer, the first and last changed offsets relative to
        the body (negative: before it) and the count of changed bytes."""
        out = []
        for part, lo in ((self.front, -self.off), (self.back, self.nbytes)):
            if torch.is_tensor(self.armed):
                bad = part != (0xFF if lo < 0 else self.armed[:part.numel()])
            elif self.armed == "pattern":
                ref = self._pat_front if lo < 0 else self._pat_back
                bad = part != ref
            else:
                bad = part != self.armed
            idx = torch.nonzero(bad).flatten()
            if idx.numel():
                first, last = int(idx[0]) + lo, int(idx[-1]) + lo
                out.append(f"{self.name}: {'front' if lo < 0 else 'back'} guard written at body offsets [{first}, {last}], "
                           f"{idx.numel()} bytes changed")
        return "; ".join(out)


def sync(device):
    if torch.device(device).type == "cuda":
        torch.cuda.synchronize(device)


def _finite(t):
    return bool(torch.isfinite(t).all()) if t.dtype.is_floating_point else True


def run_case(call, buffers, device="cuda", runs=3):
    """Run `call()` (returning a status; 0 expected) three times over `buffers` (a list of Guarded): before each run every
    buffer is prepared, after it every guard is checked.  Returns a list of problems (empty when the case is clean) and the
    last run's outputs."""
    snaps, found = [], []
    for r in range(runs):
        for g in buffers:
            g.prepare(r)
        sync(device)
        st = call()
        if st != 0:
            return [f"run {r}: status {st}"], None
        sync(device)
        found += [f"run {r}: {p}" for p in (g.problems() for g in buffers) if p]
        snaps.append({g.name: g.view().clone() for g in buffers if g.kind != "in" and g.compare})
    if runs < 3:
        return found, snaps[-1]
    za, zb, ff = snaps
    raw = lambda a: a.reshape(-1).view(torch.uint8) if a.numel() else a.reshape(-1)
    same = lambda a, b: torch.equal(raw(a), raw(b))
    for k in za:
        if same(za[k], zb[k]):
            if not same(ff[k], za[k]):
                n = int((raw(ff[k]) != raw(za[k])).sum())
                found.append(f"{k}: differs ({n} bytes) when the input guards are poisoned instead of 0: a read past an input")
        elif not _finite(ff[k]):
            found.append(f"{k}: not reproducible and not finite")
    return found, ff


def input_of(name, array, device="cuda", align=16, dtype=None, poison=0xFF):
    """An input at the end of its own guarded allocation, holding `array`."""
    a = np.ascontiguousarray(array)
    tdt = dtype or _DT[a.dtype]
    g = Guarded(name, a.nbytes, kind="in", align=align, device=device, dtype=tdt, shape=a.shape, poison=poison)
    return g.set(a)


def output_of(name, shape, dtype, device="cuda", align=16, kind="out", compare=True, guard=GUARD, pinned=False):
    n = int(np.prod(shape)) * torch.empty((), dtype=dtype).element_size()
    return Guarded(name, n, kind=kind, align=align or torch.empty((), dtype=dtype).element_size(), device=device, dtype=dtype,
                   shape=shape, compare=compare, guard=guard, pinned=pinned)
