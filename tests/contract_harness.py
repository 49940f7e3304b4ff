"""The calibrated bf16 rule of DESIGN.md §2 and the output checks shared by the kernel contract and calibration tests.

  calibrated   per slice, ||got - ref|| <= FACTOR ||arm - ref|| + FLOOR ||ref|| (+ abs_floor sqrt(count)), where the arm
               rounds to bf16 exactly where the kernel or module does; calibrated_model_rows applies it to whole tensors
  within       element by element, |got - exact| <= bound; NaN fails, an exact element passes under a zero bound
  coverage     Out (2-D, guard rows and pad columns) and Guarded (flat, guard bytes): logical elements start unwritten
               (NaN, or the dtype's guard pattern for integer dtypes), every other element holds the guard pattern and
               must keep it
  same_bits    equality of the bit patterns (tells -0 from +0, compares NaN payloads)
  reordering   two runs of the same model on the same inputs that may differ only in the order of fp32 atomic additions
               (split-K weight gradients, column sums): outputs with the same bits, every gradient within GRAD_REL x
               its scale (reordering_violations)
  periodic     operands past 2^31 bytes or elements: rows (or samples) repeat a small base block (`periodic`, the period
               checked against wrapped offsets by `no_aliasing`), every output row must have the bits of its representative
               in a small run (`same_as_representatives`), and Big outputs are scanned for coverage and guards chunk by
               chunk, with no full-size mask, clone or cast; a reduction over such an operand has no row to compare, so
               `has_power` asserts that the value a planted defect would give falls outside its bound
"""
import contextlib

import torch

FACTOR = 1.5           # DESIGN.md §2: at most 1.5 x what the rounding of the computation itself costs
FLOOR = 2.0 ** -16     # x the slice's reference norm: keeps exactly representable slices from dividing by zero
ABS_FLOOR = 4e-6       # per element, for slices whose exact value is 0 (temporal T = 1: dq = dk = 0) but whose fp32
                       # residue (dP - delta of O(1) inputs) is not; far below any rounding error of O(1e-3) outputs
LSE_TOL = 1e-4         # LSE per row: |err| <= LSE_TOL x max(1, |lse|) (fp32 from fp32 scores)
GUARD_ROWS = 3         # Out: rows past the output
PAD = 64               # Guarded: bytes before and after the output (keeps it 64-byte aligned)

# the integer view and the guard bit pattern of every dtype an output is guarded in; an integer output starts as its
# pattern, so it may only be checked for writes where no written value can equal the pattern
DTYPES = {
    torch.bfloat16: (torch.int16, 0x3F81),
    torch.float16: (torch.int16, 0x3C11),
    torch.float32: (torch.int32, 0x3F810204),
    torch.int32: (torch.int32, 0x3F810204),
    torch.int64: (torch.int64, -7777),
    torch.uint8: (torch.uint8, 0xA5),
}


def bits(t):
    return t.contiguous().view(DTYPES[t.dtype][0])


def same_bits(a, b):
    return torch.equal(bits(a), bits(b))


def _start(t):
    """Mark the logical elements of an output unwritten: NaN, or the guard pattern for integer dtypes."""
    if t.dtype.is_floating_point:
        t.fill_(float("nan"))
    else:
        t.fill_(DTYPES[t.dtype][1])


def _unwritten(t, finite):
    """Count of elements still unwritten (for floating dtypes also, with `finite`, those not finite)."""
    if t.dtype.is_floating_point:
        return int((~torch.isfinite(t.float()) if finite else torch.isnan(t)).sum())
    return int((t == DTYPES[t.dtype][1]).sum())


class Out:
    """An output of `rows` x `width` elements (row pitch ld) inside a buffer GUARD_ROWS rows longer: the logical elements
    start unwritten (or as `init`), every other element holds the guard pattern."""

    def __init__(self, dev, rows, width, dtype, ld=None, init=None):
        ld = ld or width
        self.shape = (rows + GUARD_ROWS, ld)
        self.buf = torch.empty(self.shape, dtype=dtype, device=dev)
        self.buf.view(DTYPES[dtype][0]).fill_(DTYPES[dtype][1])
        self.t = self.buf[:rows, :width]
        if init is None:
            _start(self.t)
        else:
            self.t.copy_(init)
        self.outside = torch.ones(self.shape, dtype=torch.bool, device=dev)
        self.outside[:rows, :width] = False
        self.snap = bits(self.buf).clone()

    def check(self, what):
        bad = _unwritten(self.t, finite=True)
        assert bad == 0, f"{what}: {bad} of {self.t.numel()} elements not written (still NaN) or not finite"
        moved = int((bits(self.buf) != self.snap)[self.outside].sum())
        assert moved == 0, f"{what}: {moved} elements outside the output (guard rows / pad columns) were overwritten"
        return self.t.clone()


class Guarded:
    """A tensor of `shape` inside an allocation with PAD bytes of guard pattern before and after it.  Its elements start
    unwritten or as the given init."""

    def __init__(self, dev, shape, dtype, init=None):
        n = 1
        for s in shape:
            n *= s
        self.pre = PAD // torch.empty(0, dtype=dtype).element_size()
        self.n = n
        self.buf = torch.empty(n + 2 * self.pre, dtype=dtype, device=dev)
        self.buf.view(DTYPES[dtype][0]).fill_(DTYPES[dtype][1])
        self.t = self.buf[self.pre:self.pre + n].view(shape)
        if init is None:
            _start(self.t)
        else:
            self.t.copy_(init)
        self.snap = bits(self.buf).clone()

    def guards(self, what):
        iv, sv = bits(self.buf), self.snap
        moved = int((iv[:self.pre] != sv[:self.pre]).sum() + (iv[self.pre + self.n:] != sv[self.pre + self.n:]).sum())
        assert moved == 0, f"{what}: {moved} guard elements overwritten"

    def written(self, what):
        """Guards intact and every element written (inf is a value: an f16 output may overflow)."""
        self.guards(what)
        bad = _unwritten(self.t, finite=False)
        assert bad == 0, f"{what}: {bad} of {self.n} elements not written"
        return self.t


class Report:
    """The worst value recorded per key, printed under `header` by the owning module's autouse fixture (pytest -s)."""

    def __init__(self, header, width=70, fmt="{:.3g}".format):
        self.header, self.width, self.fmt, self.worst = header, width, fmt, {}

    def record(self, key, value):
        self.worst[key] = max(self.worst[key], value) if key in self.worst else value

    def print(self):
        if self.worst:
            print("\n" + self.header)
            for k in sorted(self.worst):
                print(f"  {k:{self.width}s} {self.fmt(self.worst[k])}")


def slice_rule(key, got, ref, arm, ids, label, abs_floor=0.0):
    """Per slice (ids: slice index of every element; label(i) names slice i):
    ||got - ref|| <= FACTOR ||arm - ref|| + FLOOR ||ref|| + abs_floor sqrt(count).  A slice with no elements passes.
    Returns the worst err(got) / err(arm) (with the floor) and the message of the worst violation, or None."""
    ids = ids.reshape(-1)
    n = int(ids.max()) + 1

    def norm(x):
        return torch.zeros(n, dtype=torch.float64, device=x.device).index_add_(0, ids, x.reshape(-1) ** 2).sqrt()

    ref = ref.double()
    e_k, e_a, nrm = norm(got.double() - ref), norm(arm.double() - ref), norm(ref)
    count = torch.zeros(n, dtype=torch.float64, device=ids.device).index_add_(0, ids, torch.ones_like(ref.reshape(-1)))
    floor = FLOOR * nrm + abs_floor * count.sqrt() + (count == 0) + 1e-300
    ratio = e_k / (FACTOR * e_a + floor)
    w = int(ratio.argmax())
    measured = float((e_k / (e_a + floor)).max())
    if float(ratio[w]) <= 1.0:
        return measured, None
    return measured, (f"{key}: worst slice {label(w)}: error {float(e_k[w]):.3e} is "
                      f"{float(e_k[w] / (e_a[w] + floor[w])):.2f} x the bf16 arm's {float(e_a[w]):.3e} "
                      f"(slice norm {float(nrm[w]):.3e}; bound {FACTOR} x + {FLOOR:.1e} x norm)")


def calibrated(report, key, got, ref, arm, ids, label, abs_floor=0.0):
    """slice_rule asserted; the worst ratio is recorded under `key` and returned."""
    measured, bad = slice_rule(key, got, ref, arm, ids, label, abs_floor)
    report.record(key, measured)
    assert bad is None, bad
    return measured


def tile_slices(M, N, device):
    """Slice index [M, N] = (row // 64, col // 128): one consumer's 64 x 128 accumulator block of the GEMM, one
    warpgroup's half of a fused 128 x 128 InfoNCE tile, one 64 x 128 tile of nce.cu."""
    nc = (N + 127) // 128
    ids = (torch.arange(M, device=device)[:, None] // 64) * nc + torch.arange(N, device=device)[None, :] // 128
    return ids, lambda i: f"(row64={i // nc}, col128={i % nc})"


def within(report, key, got, exact, bound):
    """Every element: |got - exact| <= bound; NaN fails.  Records the worst |err| / bound (0 where err is 0)."""
    err = (got.double() - exact).abs()
    bad = ~(err <= bound)
    ratio = torch.where(err == 0, 0.0, err / bound)
    worst = float(ratio.max()) if ratio.numel() else 0.0
    report.record(key, worst)
    if bool(bad.any()):
        w = int(bad.reshape(-1).nonzero()[0])
        raise AssertionError(f"{key}: {int(bad.sum())} of {err.numel()} elements outside the bound, the first at flat "
                             f"index {w}: got {float(got.reshape(-1)[w]):.7e}, exact {float(exact.reshape(-1)[w]):.7e}, "
                             f"bound {float(bound.reshape(-1)[w]):.3e} (worst ratio {worst:.3g})")


def lse_check(report, tag, got, ref):
    """Per row: |lse - exact| <= LSE_TOL x max(1, |exact|)."""
    err = (got.double() - ref).abs() / ref.abs().clamp_min(1.0)
    w = int(err.reshape(-1).argmax())
    report.record(f"{tag}: lse", float(err.max()))
    assert float(err.max()) <= LSE_TOL, f"{tag}: lse: worst row (flat index {w}) relative error {float(err.max()):.3e}"


def calibrated_model_rows(tag, rows, slices=None):
    """The calibrated rule on whole tensors and, optionally, on slices of them.

    rows: (name, ours, fp32 oracle, bf16 arm, autocast run or None) per tensor.  Whole tensor: err(ours) <= 1.5 x err(arm)
    (+1e-7), both relative L2 against the fp32 oracle.  slices: name -> (ids, label) for `slice_rule` (per slice, with its
    floor of 2^-16 x the slice's norm and ABS_FLOOR).  Returns (violations, worst whole-tensor ratio, worst slice ratio),
    each ratio a (value, tensor name) pair; the autocast ratio is printed, never asserted."""
    def rel(a, b):
        return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))

    bad = []
    worst, worst_ac, worst_sl = (0.0, ""), (0.0, ""), (0.0, "")
    for name, got, ref, a, c in rows:
        e, ea = rel(got, ref), rel(a, ref)
        worst = max(worst, (e / (ea + 1e-7), name))
        if c is not None:
            worst_ac = max(worst_ac, (e / (rel(c, ref) + 1e-7), name))
        if e > FACTOR * ea + 1e-7:
            bad.append(f"{tag}: {name}: error {e:.3e} vs the bf16 oracle's {ea:.3e}")
        if slices and name in slices:
            ratio, msg = slice_rule(f"{tag}: {name}", got, ref, a, *slices[name], ABS_FLOOR)
            worst_sl = max(worst_sl, (ratio, name))
            if msg is not None:
                bad.append(msg)
    print(f"{tag}: worst err / bf16-oracle err {worst[0]:.3f} ({worst[1]})"
          + (f", worst slice {worst_sl[0]:.3f} ({worst_sl[1]})" if slices else "")
          + (f"; worst err / autocast err {worst_ac[0]:.2f} ({worst_ac[1]})" if worst_ac[1] else ""))
    return bad, worst, worst_sl


# ------------------------------------------------------------------------------ periodic operands past 2^31
CHUNK = 1 << 26         # elements per step of the scans over multi-GB outputs
WRAP = 1 << 31          # a 32-bit offset wraps (or turns negative) at a multiple of 2^31 bytes or elements


def periodic(base, rows, out=None, weights=None):
    """[rows, ...] with row r = base[r % P] (P = base.shape[0]), written by broadcast copies: nothing of the full size is
    built besides the result.  `out` (contiguous, [rows, ...]) receives it in place when given.  weights [ceil(rows / P)]
    (powers of two, so exact): period j is scaled by weights[j] in place."""
    P = base.shape[0]
    if out is None:
        out = torch.empty((rows,) + tuple(base.shape[1:]), dtype=base.dtype, device=base.device)
    full = rows // P
    w = None if weights is None else weights.to(base.dtype).to(base.device)
    if full:
        body = out[:full * P].view((full,) + tuple(base.shape))
        body.copy_(base)
        if w is not None:
            body.mul_(w[:full].view((full,) + (1,) * base.dim()))
    if rows > full * P:
        out[full * P:rows].copy_(base[:rows - full * P])
        if w is not None:
            out[full * P:rows].mul_(w[full])
    return out


def no_aliasing(name, period_rows, row_elems, elsize, nbytes):
    """The displacement rule: in a buffer of `nbytes` whose rows of `row_elems` elements (`elsize` bytes each) repeat every
    `period_rows` rows, a move by a multiple of 2^31 bytes (and so of 2^32) must never land on an element of the same
    residue and column, i.e. must not be a multiple of one period.  Otherwise an offset that wrapped would read or write
    the very value a correct one does, and no comparison could see it."""
    period = period_rows * row_elems * elsize
    for k in range(1, nbytes // WRAP + 1):
        assert (k * WRAP) % period != 0, (f"{name}: a period of {period_rows} rows x {row_elems} elements ({period} bytes) "
                                          f"divides {k} x 2^31 bytes: a wrapped offset would alias onto its own residue")


def crossing(report, case, name, t, claim):
    """Assert that tensor t (the logical operand) reaches past `claim`, one of '2^31 bytes', '2^32 bytes', '2^31 elements',
    at its largest byte or element offset; records the largest offset / the boundary."""
    last = t.numel() - 1
    off, bound = {"2^31 bytes": (last * t.element_size(), 1 << 31), "2^32 bytes": (last * t.element_size(), 1 << 32),
                  "2^31 elements": (last, 1 << 31)}[claim]
    report.record(f"{case}: {name} past {claim} (largest offset / boundary)", off / bound)
    assert off >= bound, f"{case}: {name} reaches offset {off}, short of {claim}: the case no longer tests what it claims"


def same_as_representatives(what, big, rep, chunk=CHUNK):
    """Every row r of big ([rows, ...]) has the bits of rep[r % P] (rep [P, ...]), compared over whole periods at about
    `chunk` elements a step.  The message names the first differing row, its residue and its first differing column."""
    P = rep.shape[0]
    rb = bits(rep).reshape(P, -1)
    per = rb.shape[1]
    step = max(1, chunk // (P * per)) * P
    rows = big.shape[0]
    for r0 in range(0, rows, step):
        n = min(step, rows - r0)
        g = bits(big[r0:r0 + n]).reshape(n, per)
        full = n // P
        diff = torch.empty(n, dtype=torch.bool, device=g.device)
        if full:
            diff[:full * P] = (g[:full * P].view(full, P, per) != rb).any(-1).view(-1)
        if n > full * P:
            diff[full * P:] = (g[full * P:] != rb[:n - full * P]).any(-1)
        if bool(diff.any()):
            r = int(diff.nonzero()[0])
            c = int((g[r] != rb[(r0 + r) % P]).nonzero()[0])
            raise AssertionError(f"{what}: {int(diff.sum())} rows of [{r0}, {r0 + n}) differ from their representatives, "
                                 f"the first row {r0 + r} (residue {(r0 + r) % P}) at flat column {c}")


def has_power(report, key, exact, planted, bound):
    """The self-check of a reduction over a periodic operand: the value a planted defect gives (rows past a boundary
    dropped, or read from the wrong place) must fall outside the bound at every element, or the check could not see that
    defect.  Records the largest bound / |planted - exact|, which is below 1 when the check has power everywhere."""
    gap = (planted.double() - exact.double()).abs()
    ratio = bound.double() / gap
    worst = float(ratio.max())
    report.record(f"{key}: self-check, largest bound / |planted - exact|", worst)
    assert worst < 1.0, (f"{key}: the planted defect stays inside the bound at {int((ratio >= 1).sum())} of {ratio.numel()} "
                         f"elements (worst bound / gap {worst:.3g}): this check cannot see it")


class Big:
    """A multi-GB output of `shape` inside one allocation with PAD bytes of guard pattern before and after it.  Its elements
    start unwritten (NaN, or the pattern for integer dtypes); `check` scans it in chunks of about CHUNK elements for
    unwritten or non-finite elements and checks the guards against the pattern, without a full-size mask, clone or cast."""

    def __init__(self, dev, shape, dtype, chunk=CHUNK):
        n = 1
        for s in shape:
            n *= s
        self.pre, self.n, self.chunk = PAD // torch.empty(0, dtype=dtype).element_size(), n, chunk
        self.buf = torch.empty(n + 2 * self.pre, dtype=dtype, device=dev)
        iv = self.buf.view(DTYPES[dtype][0])
        iv[:self.pre].fill_(DTYPES[dtype][1])
        iv[self.pre + n:].fill_(DTYPES[dtype][1])
        self.t = self.buf[self.pre:self.pre + n].view(shape)
        _start(self.t)

    def guards(self, what):
        iv, pat = self.buf.view(DTYPES[self.buf.dtype][0]), DTYPES[self.buf.dtype][1]
        for side, g in (("before", iv[:self.pre]), ("after", iv[self.pre + self.n:])):
            moved = int((g != pat).sum())
            assert moved == 0, f"{what}: {moved} guard elements {side} the output overwritten"

    def check(self, what):
        """Guards intact and every element written and finite; returns the output."""
        self.guards(what)
        pat = DTYPES[self.buf.dtype][1]
        flat = self.buf[self.pre:self.pre + self.n]
        for i in range(0, self.n, self.chunk):
            c = flat[i:i + self.chunk]
            bad = ~torch.isfinite(c) if c.dtype.is_floating_point else c == pat
            if bool(bad.any()):
                raise AssertionError(f"{what}: {int(bad.sum())} elements of [{i}, {i + c.numel()}) not written or not "
                                     f"finite, the first at flat index {i + int(bad.nonzero()[0])}")
        return self.t


GRAD_REL = 1e-5         # max |g - g_ref| <= GRAD_REL x scale: split-K atomics reorder (about 1e-7 between runs)


def grad_scale(grads, n):
    """max |g| of gradient n.  k_proj.bias is measured against its layer's whole q/k/v bias gradient: its exact value is zero
    (a key bias shifts every logit of a query row equally), so what the kernels compute is the rounding residue of a column
    sum that cancels, accumulated with fp32 atomics, and its own maximum is that residue."""
    if n.endswith("self_attn.k_proj.bias"):
        return max(float(grads[n.replace("k_proj", p)].abs().max()) for p in ("q_proj", "k_proj", "v_proj"))
    return float(grads[n].abs().max())


def reordering_violations(ref_out, got_out, ref_grads, got_grads, rel=GRAD_REL):
    """Two runs that may differ only in the order of fp32 atomic additions.  ref_out / got_out: {name: tensor}, which must
    be finite and have the same bits; ref_grads / got_grads: {name: tensor or None}, the same names receiving a gradient
    and max |got - ref| <= rel x grad_scale(ref_grads, name) for each.  Returns (violations, (worst |got - ref| / scale,
    its name)); the worst ratio is over the gradients."""
    bad = []
    for n, r in ref_out.items():
        g = got_out[n]
        if not bool(torch.isfinite(g.float()).all()):
            bad.append(f"{n}: not finite")
        elif not same_bits(r, g):
            d = float((g.double() - r.double()).abs().max())
            bad.append(f"{n}: bits differ (max |difference| {d:.3e})")
    if set(ref_grads) != set(got_grads):
        bad.append(f"gradients on one side only: {sorted(set(ref_grads) ^ set(got_grads))}")
    worst = (0.0, None)
    for n in sorted(set(ref_grads) & set(got_grads)):
        r, g = ref_grads[n], got_grads[n]
        if (r is None) != (g is None):
            bad.append(f"{n}: gradient {'missing' if g is None else 'unexpected'}")
            continue
        if r is None:
            continue
        scale = grad_scale(ref_grads, n)
        diff = float((g.double() - r.double()).abs().max())
        if not diff <= rel * scale:          # NaN fails
            bad.append(f"{n}: max |difference| {diff:.3e} > {rel:.0e} x scale {scale:.3e}")
        if scale > 0 and diff / scale > worst[0]:
            worst = (diff / scale, n)
    return bad, worst


@contextlib.contextmanager
def no_tf32():
    """The fp32 oracle is the truth: no TF32 in its matmuls or convolutions."""
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved
