"""The shared rule and output checks of contract_harness.py at their boundaries, on the CPU: the calibrated slice rule at
exactly FACTOR x the arm, the absolute floor, empty slices, the element check on NaN and zero bounds, write coverage and
guard elements for every guarded dtype, and bitwise comparison of signed zeros."""
import pytest
import torch

from contract_harness import ABS_FLOOR, DTYPES, FACTOR, FLOOR, Guarded, Out, Report, calibrated, same_bits, within

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
