"""The shared rule and output checks of contract_harness.py at their boundaries, on the CPU: the calibrated slice rule at
exactly FACTOR x the arm, the absolute floor, empty slices, the element check on NaN and zero bounds, write coverage and
guard elements for every guarded dtype, bitwise comparison of signed zeros, and the reordering rule of two runs that differ
only in the order of fp32 atomic additions."""
import pytest
import torch

from contract_harness import (ABS_FLOOR, DTYPES, FACTOR, FLOOR, GRAD_REL, Guarded, Out, Report, calibrated,
                              reordering_violations, same_bits, within)

F64 = torch.float64


def _label(i):
    return f"slice {i}"


def test_slice_at_exactly_factor_times_the_arm_passes_and_just_above_fails():
    """Slice 1 has reference norm 1 and arm error 1: its bound is FACTOR + FLOOR exactly.  Slice 0's large arm error must
    not lend slice 1 any of its allowance."""
    ids = torch.tensor([0, 0, 1, 1])
    ref = torch.tensor([1.0, 0.0, 1.0, 0.0], dtype=F64)
    arm = ref + torch.tensor([0.0, 100.0, 0.0, 1.0], dtype=F64)
    bound = FACTOR * 1.0 + FLOOR
    at = ref + torch.tensor([0.0, 0.0, 0.0, bound], dtype=F64)
    report = Report("test")
    calibrated(report, "at", at, ref, arm, ids, _label)
    assert report.worst["at"] == pytest.approx(bound / (1.0 + FLOOR))
    above = ref + torch.tensor([0.0, 0.0, 0.0, bound * (1 + 2.0 ** -40)], dtype=F64)
    with pytest.raises(AssertionError, match="slice 1"):
        calibrated(Report("test"), "above", above, ref, arm, ids, _label)


def test_abs_floor_admits_fp32_residue_on_a_zero_reference_only_when_asked():
    ids = torch.zeros(64, dtype=torch.long)
    ref = torch.zeros(64, dtype=F64)
    got = torch.full((64,), 1e-7, dtype=F64)          # fp32-sized residue where the exact value and the arm are 0
    calibrated(Report("test"), "with abs_floor", got, ref, ref, ids, _label, ABS_FLOOR)
    with pytest.raises(AssertionError):
        calibrated(Report("test"), "without", got, ref, ref, ids, _label)


def test_an_empty_slice_passes():
    ids = torch.tensor([0, 0, 2, 2])                  # slice 1 has no elements
    ref = torch.tensor([1.0, 2.0, 3.0, 4.0], dtype=F64)
    arm = ref + 1e-3
    for abs_floor in (0.0, ABS_FLOOR):
        assert calibrated(Report("test"), "empty", ref + 1e-3, ref, arm, ids, _label, abs_floor) <= 1.0


def test_within_fails_on_nan_and_passes_an_exact_element_under_a_zero_bound():
    exact = torch.tensor([1.0, 2.0, 0.0], dtype=F64)
    bound = torch.tensor([1e-3, 1e-3, 0.0], dtype=F64)
    report = Report("test")
    within(report, "exact", exact.float(), exact, bound)
    assert report.worst["exact"] == 0.0
    with pytest.raises(AssertionError):
        within(report, "nan", torch.tensor([1.0, float("nan"), 0.0]), exact, bound)
    with pytest.raises(AssertionError):
        within(report, "over", torch.tensor([1.0, 2.0, 1e-30]), exact, bound)


DT = list(DTYPES)
DT_IDS = [str(d).replace("torch.", "") for d in DT]


def _value(dtype):
    """A value no output starts as: not NaN and not the guard pattern."""
    return 1.5 if dtype.is_floating_point else 7


@pytest.mark.parametrize("dtype", DT, ids=DT_IDS)
def test_out_catches_an_unwritten_element_and_an_overwritten_guard(dtype):
    def written(ld=None):
        o = Out("cpu", 4, 8, dtype, ld=ld)
        o.t.fill_(_value(dtype))
        return o
    assert same_bits(written(ld=12).check("all written"), torch.full((4, 8), _value(dtype), dtype=dtype))
    o = Out("cpu", 4, 8, dtype)
    o.t[:, 1:].fill_(_value(dtype))
    with pytest.raises(AssertionError, match="not written"):
        o.check("one column unwritten")
    o = written()
    o.buf[4, 0] = _value(dtype)                       # a guard row
    with pytest.raises(AssertionError, match="overwritten"):
        o.check("guard row")
    o = written(ld=12)
    o.buf[2, 9] = _value(dtype)                       # a pad column
    with pytest.raises(AssertionError, match="overwritten"):
        o.check("pad column")


@pytest.mark.parametrize("dtype", DT, ids=DT_IDS)
def test_guarded_catches_an_unwritten_element_and_an_overwritten_guard(dtype):
    g = Guarded("cpu", (3, 5), dtype)
    g.t.fill_(_value(dtype))
    g.written("all written")
    g.t[2, 4] = Guarded("cpu", (1,), dtype).t[0]      # its start value: unwritten
    with pytest.raises(AssertionError, match="not written"):
        g.written("one unwritten")
    for where in (0, -1):                             # before and after the tensor
        g = Guarded("cpu", (3, 5), dtype)
        g.t.fill_(_value(dtype))
        g.buf[where] = _value(dtype)
        with pytest.raises(AssertionError, match="guard"):
            g.guards("guard")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
def test_same_bits_tells_signed_zeros_apart(dtype):
    pos, neg = torch.zeros(3, dtype=dtype), torch.zeros(3, dtype=dtype)
    neg[1] = -0.0
    assert bool((pos == neg).all()) and not same_bits(pos, neg)
    assert same_bits(neg, neg.clone())


def _layer_grads(seed=0):
    g = torch.Generator().manual_seed(seed)
    pre = "clipmodel.vision_model.encoder.layers.0.self_attn."
    grads = {pre + f"{n}.bias": torch.randn(8, generator=g) for n in ("q_proj", "k_proj", "v_proj")}
    grads[pre + "k_proj.bias"] *= 1e-4                # the cancelling key bias: a rounding residue
    grads[pre + "out_proj.weight"] = torch.randn(8, 8, generator=g)
    grads["clipmodel.text_model.embeddings.token_embedding.weight"] = None
    return pre, grads


def test_reordering_rule_flags_1e4_passes_1e7_and_scales_k_bias_by_qkv():
    pre, ref = _layer_grads()
    out = {"loss": torch.tensor(1.25), "vis": torch.randn(4, 8, generator=torch.Generator().manual_seed(1))}
    w = pre + "out_proj.weight"
    scale = float(ref[w].abs().max())
    for rel, flagged in ((1e-4, True), (1e-7, False)):
        got = dict(ref)
        got[w] = ref[w].clone()
        got[w][3, 5] += rel * scale
        bad, worst = reordering_violations(out, {k: v.clone() for k, v in out.items()}, ref, got)
        assert bool(bad) == flagged and (not bad or w in bad[0]), bad
        assert worst[1] == w and worst[0] == pytest.approx(rel, rel=0.1)     # fp32 rounding of the planted add
    # k_proj.bias: a difference of 1e-6 x the q/k/v maximum passes although it is ~1e-2 of its own maximum, and 1e-4 of
    # the q/k/v maximum fails
    k = pre + "k_proj.bias"
    qkv = max(float(ref[pre + f"{n}.bias"].abs().max()) for n in ("q_proj", "k_proj", "v_proj"))
    assert float(ref[k].abs().max()) < 1e-3 * qkv
    for rel, flagged in ((1e-6, False), (1e-4, True)):
        got = dict(ref)
        got[k] = ref[k] + rel * qkv
        bad, worst = reordering_violations(out, out, ref, got)
        assert bool(bad) == flagged, bad
        assert worst[1] == k and worst[0] == pytest.approx(rel, rel=1e-3)
    assert GRAD_REL == 1e-5


def test_reordering_rule_wants_the_same_output_bits_and_the_same_gradients():
    _, ref = _layer_grads()
    out = {"loss": torch.tensor(0.0), "vis": torch.ones(2, 3)}
    neg = {"loss": torch.tensor(-0.0), "vis": torch.ones(2, 3)}
    bad, _ = reordering_violations(out, neg, ref, ref)
    assert len(bad) == 1 and bad[0].startswith("loss: bits differ"), bad
    nan = {"loss": torch.tensor(0.0), "vis": torch.full((2, 3), float("nan"))}
    assert reordering_violations(nan, nan, ref, ref)[0] == ["vis: not finite"]
    name = "clipmodel.text_model.embeddings.token_embedding.weight"
    assert any(name in b for b in reordering_violations(out, out, ref, dict(ref, **{name: torch.zeros(2)}))[0])
    nang = {k: (None if v is None else v.clone()) for k, v in ref.items()}
    w = next(k for k in ref if k.endswith("out_proj.weight"))
    nang[w][0, 0] = float("nan")
    assert any(w in b for b in reordering_violations(out, out, ref, nang)[0])
    assert reordering_violations(out, out, ref, {k: v for k, v in ref.items() if k != w})[0]


# ------------------------------------------------------------------ periodic operands past 2^31 (small, tiny chunks)
from contract_harness import WRAP, Big, crossing, no_aliasing, periodic, same_as_representatives  # noqa: E402


def _periodic_case(rows=999, P=7, W=24, dtype=torch.bfloat16):
    base = torch.randn(P, W, generator=torch.Generator().manual_seed(P)).to(dtype)
    return base, periodic(base, rows)


def test_periodic_builder_repeats_the_base_with_a_partial_tail_and_fills_in_place():
    base, big = _periodic_case()
    want = base.repeat(999 // 7 + 1, 1)[:999]
    assert same_bits(big, want)
    out = torch.full((999, 24), float("nan"), dtype=torch.bfloat16)
    assert periodic(base, 999, out=out) is out and same_bits(out, want)
    assert same_bits(periodic(base, 5), base[:5])            # fewer rows than one period


def test_displacement_rule_refuses_a_period_that_divides_2e31_bytes():
    no_aliasing("GEMM 41 x 128 rows", 41 * 128, 3072, 2, 803_328 * 3072 * 2)      # 2^17 x 123 bytes: never divides
    no_aliasing("below 2^31: nothing to wrap", 128, 1024, 2, WRAP - 1)
    with pytest.raises(AssertionError, match="divides 1 x 2"):
        no_aliasing("128 rows x 1024", 128, 1024, 2, WRAP + 1)                     # 2^18 bytes divides 2^31
    with pytest.raises(AssertionError, match="divides 2 x 2"):
        no_aliasing("2^32 bytes", 1, 1 << 30, 4, 2 * WRAP)                         # divides 2^32, not 2^31


def test_big_coverage_scan_finds_a_nan_in_the_last_chunk_and_both_guards():
    b = Big("cpu", (10, 7), torch.bfloat16, chunk=16)                              # 70 elements: the last chunk holds 6
    b.t.fill_(1.0)
    assert b.check("all written") is b.t
    b.t.view(-1)[-1] = float("nan")
    with pytest.raises(AssertionError, match=r"\[64, 70\).*flat index 69"):
        b.check("last")
    b.t.fill_(float("inf"))
    with pytest.raises(AssertionError, match="not finite"):
        b.check("inf")
    b.t.fill_(1.0)
    b.buf.view(torch.int16)[b.pre - 1] = 0
    with pytest.raises(AssertionError, match="before"):
        b.check("guard before")
    b.buf.view(torch.int16)[b.pre - 1] = DTYPES[torch.bfloat16][1]
    b.buf.view(torch.int16)[b.pre + b.n] = 0
    with pytest.raises(AssertionError, match="after"):
        b.check("guard after")


def test_big_starts_unwritten_for_an_integer_dtype():
    b = Big("cpu", (5,), torch.int32, chunk=2)
    with pytest.raises(AssertionError, match="not written"):
        b.check("int32")
    b.t.fill_(3)
    b.check("int32")


def test_representatives_catch_a_block_moved_by_a_multiple_of_2e31_bytes_modulo_the_buffer():
    """The block of rows a wrapped offset would write: the data of the position k x 2^31 bytes further on, taken modulo the
    buffer's size.  The period keeps that move off the element's own residue and column, so the block differs."""
    base, big = _periodic_case()
    same_as_representatives("clean", big, base, chunk=100)
    flat = big.view(-1)
    n = flat.numel()
    for k in (1, 2, 3):
        d = (k * WRAP // 2) % n                                                  # elements (bf16)
        assert d % (7 * 24) != 0
        bad = big.clone()
        rows = torch.arange(400 * 24, 410 * 24)
        bad.view(-1)[rows] = flat[(rows + d) % n]
        with pytest.raises(AssertionError, match=r"row 40\d \(residue"):
            same_as_representatives(f"moved by {k} x 2^31 bytes", bad, base, chunk=100)


def test_representatives_catch_a_sample_that_read_its_neighbour():
    B, P, S, W = 8, 3, 5, 16
    base = torch.randn(P, S * W, generator=torch.Generator().manual_seed(1))
    big = periodic(base, B)
    same_as_representatives("clean", big, base, chunk=64)
    big[4] = big[5]
    with pytest.raises(AssertionError, match="first row 4 \\(residue 1\\)"):
        same_as_representatives("neighbour", big, base, chunk=64)
    big = periodic(base, B)
    big[7, 3] = -big[7, 3]                                                       # the partial last period
    with pytest.raises(AssertionError, match="row 7 .*column 3"):
        same_as_representatives("tail", big, base, chunk=64)


def test_crossing_claims_are_checked_on_the_operands_extent():
    report = Report("test")
    huge = torch.zeros(1, dtype=torch.bfloat16).expand((1 << 31) + 1)            # no memory behind it
    crossing(report, "case", "x", huge, "2^31 elements")
    crossing(report, "case", "x", huge, "2^32 bytes")
    assert report.worst["case: x past 2^31 elements (largest offset / boundary)"] == 1.0
    with pytest.raises(AssertionError, match="short of 2\\^31 elements"):
        crossing(report, "case", "y", huge[:1 << 31], "2^31 elements")
    with pytest.raises(AssertionError, match="short of 2\\^31 bytes"):
        crossing(report, "case", "z", huge[:1 << 30], "2^31 bytes")


def test_periodic_builder_scales_each_period_by_its_weight():
    from oracle.gemm_ref import block_weights
    base, _ = _periodic_case()
    w = block_weights((999 + 6) // 7)
    big = periodic(base, 999, weights=w)
    want = torch.stack([base[r % 7] * w[r // 7].to(torch.bfloat16) for r in range(999)])
    assert same_bits(big, want)


def test_has_power_fails_when_a_planted_defect_stays_inside_the_bound():
    from contract_harness import has_power
    report = Report("test")
    exact = torch.tensor([10.0, -10.0], dtype=F64)
    has_power(report, "k", exact, exact * 0.9, torch.tensor([0.5, 0.5], dtype=F64))
    assert report.worst["k: self-check, largest bound / |planted - exact|"] == pytest.approx(0.5)
    with pytest.raises(AssertionError, match="1 of 2 elements"):
        has_power(report, "weak", exact, torch.tensor([9.0, -9.9], dtype=F64), torch.tensor([0.5, 0.5], dtype=F64))
