"""H100: the optimizer kernels (optim.cu) against oracle/optim_ref.py, pinned on the CPU by test_embed_reference_cpu.py.

Tables are built here row by row (per-tensor step_size and decay, decay 0 for the no-decay groups), and every tensor is a
view into a larger allocation whose guard elements hold a fixed bit pattern.

  norm       within optim_ref's derived bound of the float64 norm; bitwise repeatable across calls and tables; the clip
             coefficient bit-exact from the kernel's norm; zero gradients and max_norm <= 0 give 1; NaN / inf gradients
             give torch.nn.utils.clip_grad_norm_'s outcome
  step       every element of p, m, v within the bound after each of 3 steps; the bf16 target is p.to(bf16) bit for bit
  paths      p, g, m, v or the bf16 target misaligned on its own drops its chunks to the scalar loop: same bits
  cast       xp_cast_table bit-exact for bf16 and fp32-copy rows
  coverage   guard elements untouched after the norm, the scaling, the step and the cast
  refusals   betas outside [0, 1), eps < 0, an empty block map: refused before any launch
"""
import math

import numpy as np
import pytest
import torch

from contract_harness import DTYPES, Report, bits, within
from oracle import optim_ref as O

pytestmark = pytest.mark.gpu

bf16, f32 = torch.bfloat16, torch.float32
GUARD = 16                     # fp32 guard elements on each side of every tensor (64 bytes)
SIZES = [1, 2, 3, 4, 5, 8191, 8192, 8193, 3 * 8192 + 77]
BETAS, EPS = (0.9, 0.98), 1e-6
REPORT = Report("optim: worst |err| / bound", width=40)


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda", 0)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    REPORT.print()


def _lib():
    from xpretrain_b200 import _lib
    return _lib


def _ops():
    from xpretrain_b200 import ops
    return ops


class Slot:
    """n elements of `dtype` at element offset `off` past a 64-byte boundary, GUARD pattern elements on each side."""

    def __init__(self, dev, n, dtype=f32, off=0, init=None):
        self.buf = torch.empty(n + off + 2 * GUARD, dtype=dtype, device=dev)
        bits(self.buf).fill_(DTYPES[dtype][1])
        self.lo, self.n = GUARD + off, n
        self.t = self.buf[self.lo:self.lo + n]
        if init is not None:
            self.t.copy_(init)
        self.snap = bits(self.buf).clone()

    def guards_intact(self):
        b, s = bits(self.buf), self.snap
        return torch.equal(b[:self.lo], s[:self.lo]) and torch.equal(b[self.lo + self.n:], s[self.lo + self.n:])


class Set:
    """Tensors p, g, m, v (+ bf16 target) for `sizes`, seeded; `mis` names the one operand to misalign by one element."""

    def __init__(self, dev, sizes, seed, mis=None, bf16_target=True, grads=None):
        g = torch.Generator(device=dev).manual_seed(seed)
        self.sizes = sizes
        self.rows = []
        for i, n in enumerate(sizes):
            p = torch.randn(n, generator=g, device=dev)
            gr = torch.randn(n, generator=g, device=dev) * (0.01 if i % 3 == 0 else 1.0) if grads is None else grads[i]
            m = torch.randn(n, generator=g, device=dev) * 0.01
            v = torch.rand(n, generator=g, device=dev) * 1e-4
            r = {k: Slot(dev, n, off=1 if mis == k else 0, init=x) for k, x in (("p", p), ("g", gr), ("m", m), ("v", v))}
            r["pb"] = Slot(dev, n, bf16, off=1 if mis == "pb" else 0) if bf16_target else None
            r["step_size"] = O.f32(O.step_size_of(3e-4 * (1 + i % 2), BETAS, 1))
            r["decay"] = 0.0 if i % 4 == 1 else O.f32(3e-4 * 0.05)          # decay 0: the no-decay groups
            self.rows.append(r)
        self.tab = _ops().OptTable(list(sizes), dev)
        self.fill()

    def fill(self, step_sizes=None):
        rows = self.tab.begin()
        for k in ("p", "g", "m", "v"):
            rows[k] = [r[k].t.data_ptr() for r in self.rows]
        rows["p_bf16"] = [r["pb"].t.data_ptr() if r["pb"] is not None else 0 for r in self.rows]
        rows["step_size"] = [r["step_size"] for r in self.rows]
        rows["decay"] = [r["decay"] for r in self.rows]
        self.tab.upload()

    def args(self):
        return self.tab.launch_args

    def norm(self, max_norm):
        _ops().opt_grad_norm(self.tab, max_norm)
        return self.tab.norm.clone()

    def scale(self):
        _ops().opt_scale_grads(self.tab)

    def step(self, with_norm=True):
        _ops().opt_adamw_step(self.tab, BETAS[0], BETAS[1], EPS, clip=with_norm)

    def snapshot(self):
        return [{k: r[k].t.clone() for k in ("p", "g", "m", "v")} for r in self.rows]

    def guards_intact(self):
        return all(r[k].guards_intact() for r in self.rows for k in ("p", "g", "m", "v", "pb") if r[k] is not None)


def check_norm(s, got):
    norm, rel = O.grad_norm_ref([r["g"].t for r in s.rows])
    err = abs(float(got[0]) - norm)
    REPORT.record("grad_norm (relative)", err / (rel * norm))
    assert err <= rel * norm, f"norm {float(got[0])} vs {norm}: {err / norm:.3g} relative (bound {rel:.3g})"


# ============================================================================================== norm
@pytest.mark.parametrize("mis", [None, "g"])
def test_grad_norm_within_bound_and_repeatable(dev, mis):
    s = Set(dev, SIZES, seed=1, mis=mis)
    a = s.norm(1.0)
    check_norm(s, a)
    assert float(a[1]) == O.clip_coef_f32(1.0, float(a[0]))
    b = s.norm(1.0)
    fresh = Set(dev, SIZES, seed=1, mis=mis)
    c = fresh.norm(1.0)
    assert torch.equal(bits(a), bits(b)) and torch.equal(bits(a), bits(c)), "the norm is not bitwise repeatable"
    assert s.guards_intact()


def test_grad_norm_edges(dev):
    zero = Set(dev, [5, 8193], seed=2, grads=[torch.zeros(5, device=dev), torch.zeros(8193, device=dev)])
    nz = zero.norm(1.0)
    assert float(nz[0]) == 0.0 and float(nz[1]) == 1.0
    s = Set(dev, [5, 8193], seed=3)
    for mx in (0.0, -1.0):
        assert float(s.norm(mx)[1]) == 1.0
    assert float(s.norm(1e30)[1]) == 1.0


@pytest.mark.parametrize("bad", [float("nan"), float("inf")])
def test_non_finite_gradient_matches_clip_grad_norm(dev, bad):
    grads = [torch.randn(n, device=dev) for n in (7, 8193)]
    grads[1][4000] = bad
    s = Set(dev, [7, 8193], seed=4, grads=[g.clone() for g in grads])
    got = s.norm(1.0)
    s.scale()
    params = [torch.nn.Parameter(torch.zeros_like(g)) for g in grads]
    for p, g in zip(params, grads):
        p.grad = g.clone()
    total = torch.nn.utils.clip_grad_norm_(params, 1.0, foreach=False)
    assert (math.isnan(float(got[0])) and math.isnan(float(total))) or float(got[0]) == float(total)
    for r, p in zip(s.rows, params):
        a, b = r["g"].t, p.grad
        assert torch.equal(torch.isnan(a), torch.isnan(b)) and torch.equal(a[~torch.isnan(a)], b[~torch.isnan(b)])
    assert s.guards_intact()


def test_scale_only(dev):
    s = Set(dev, SIZES, seed=5)
    before = [r["g"].t.clone() for r in s.rows]
    n = s.norm(1e6)                                     # coef 1: the gradients keep their bits
    assert float(n[1]) == 1.0
    s.scale()
    assert all(torch.equal(bits(r["g"].t), bits(b)) for r, b in zip(s.rows, before))
    n = s.norm(0.5)
    coef = float(n[1])
    assert coef < 1.0
    s.scale()
    for r, b in zip(s.rows, before):
        assert torch.equal(bits(r["g"].t), bits(b * torch.tensor(coef, device=dev)))     # one IEEE fp32 product
    assert s.guards_intact()


# ============================================================================================== step
def _check_step(tag, s, before, coef):
    for i, (r, b) in enumerate(zip(s.rows, before)):
        ref = O.adamw_ref(b["p"], b["g"], b["m"], b["v"], coef, BETAS[0], BETAS[1], EPS, r["step_size"], r["decay"])
        for k in ("p", "m", "v"):
            within(REPORT, f"adamw {k}", r[k].t, *ref[k])
        assert float(ref["p"][1].max()) < 1e-2 * r["step_size"]
        if r["pb"] is not None:
            assert torch.equal(bits(r["pb"].t), bits(r["p"].t.to(bf16))), f"{tag}: bf16 target of tensor {i}"


@pytest.mark.parametrize("clip", [True, False])
def test_adamw_steps_within_bound(dev, clip):
    s = Set(dev, SIZES, seed=6)
    for step in range(1, 4):
        for r in s.rows:
            r["step_size"] = O.f32(O.step_size_of(3e-4, BETAS, step))
        s.fill()
        before = s.snapshot()
        coef = 1.0
        if clip:
            coef = float(s.norm(0.5)[1])
            assert coef < 1.0
        s.step(with_norm=clip)
        _check_step(f"step {step}", s, before, coef)
    assert s.guards_intact()


@pytest.mark.parametrize("mis", ["p", "g", "m", "v", "pb"])
def test_misaligned_operand_takes_the_scalar_path_with_the_same_bits(dev, mis):
    a, b = Set(dev, SIZES, seed=7), Set(dev, SIZES, seed=7, mis=mis)
    assert all(r[mis].t.data_ptr() % 16 != 0 for r in b.rows)
    for s in (a, b):
        s.norm(0.5)
        b.tab.norm.copy_(a.tab.norm)                 # the same coefficient (the norm itself may differ in order)
        s.step()
    for ra, rb in zip(a.rows, b.rows):
        for k in ("p", "m", "v", "pb"):
            assert torch.equal(bits(ra[k].t), bits(rb[k].t)), f"{mis} misaligned: {k} differs"
    assert b.guards_intact()


def test_model_sized_table(dev):
    """~300 tensors with CLIP-ViP B/16's parameter sizes (12 + 12 layers of 768 / 512 wide), one table."""
    sizes = []
    for C, layers in ((768, 12), (512, 12)):
        for _ in range(layers):
            sizes += [C * C, C] * 4 + [4 * C * C, 4 * C, 4 * C * C, C] + [C] * 4
    sizes += [50 + 1, 768, 197 * 768, 768 * 768 * 3 // 4, 12 * 768, 3 * 768, 49408 * 512 // 8, 77 * 512, 512, 512,
              512 * 512, 768 * 512]
    assert 290 <= len(sizes) <= 400
    s = Set(dev, sizes, seed=8, bf16_target=False)
    before = s.snapshot()
    check_norm(s, s.norm(1.0))
    coef = float(s.tab.norm[1])
    s.step()
    _check_step("model table", s, before, coef)
    assert s.guards_intact()


def test_cast_table_is_exact(dev):
    ops = _ops()
    sizes = [1, 5, 8192, 8193, 3 * 8192 + 77]
    src = [torch.randn(n, device=dev) * 100 for n in sizes]
    dst = [Slot(dev, n, bf16 if i % 2 == 0 else f32, off=i % 3) for i, n in enumerate(sizes)]
    tab = ops.OptTable(sizes, dev)
    rows = tab.begin()
    rows["g"] = [x.data_ptr() for x in src]
    rows["p_bf16"] = [d.t.data_ptr() if d.t.dtype == bf16 else 0 for d in dst]
    rows["p"] = [d.t.data_ptr() if d.t.dtype == f32 else 0 for d in dst]
    tab.upload()
    ops.cast_table(tab)
    for x, d in zip(src, dst):
        assert torch.equal(bits(d.t), bits(x.to(d.t.dtype))) and d.guards_intact()


# ============================================================================================== refusals
@pytest.mark.parametrize("b1,b2,eps", [(1.0, 0.98, 1e-6), (0.9, 1.0, 1e-6), (-0.1, 0.98, 1e-6), (0.9, -0.5, 1e-6),
                                       (0.9, 0.98, -1e-6), (float("nan"), 0.98, 1e-6)])
def test_adamw_refuses_bad_hyperparameters_before_any_launch(dev, b1, b2, eps):
    lib = _lib().lib()
    s = Set(dev, [5], seed=9)
    before = s.snapshot()
    n0 = int(lib.xp_launch_count())
    t, bm, nb = s.args()
    assert lib.xp_opt_adamw_step(t, bm, nb, None, b1, b2, eps, torch.cuda.current_stream().cuda_stream) != 0
    assert int(lib.xp_launch_count()) == n0
    assert all(torch.equal(bits(r["p"].t), bits(b["p"])) for r, b in zip(s.rows, before))


def test_empty_block_map_is_refused(dev):
    lib = _lib().lib()
    s = Set(dev, [5], seed=10)
    t, bm, _ = s.args()
    st = torch.cuda.current_stream().cuda_stream
    n0 = int(lib.xp_launch_count())
    assert lib.xp_opt_grad_norm(t, bm, 0, s.tab.partial.data_ptr(), 1.0, s.tab.norm.data_ptr(), st) != 0
    assert lib.xp_opt_scale_grads(t, bm, 0, s.tab.norm.data_ptr(), st) != 0
    assert lib.xp_opt_adamw_step(t, bm, 0, None, 0.9, 0.98, 1e-6, st) != 0
    assert lib.xp_cast_table(t, bm, 0, st) != 0
    assert int(lib.xp_launch_count()) == n0
