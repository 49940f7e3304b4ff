"""CPU: the vectorised row kernels refuse misaligned operands on the host, before any CUDA call.

Every entry point of rowops.cu whose kernel moves 16-byte vectors is called through the C ABI with fabricated pointer
values (never dereferenced) and rows = 0, one operand misaligned at a time: the call must fail with a message naming that
operand and the alignment.  The same call with every operand aligned must get past those checks, to the CUDA driver (no
GPU: "CUDA driver unavailable"; on a GPU machine, rows = 0 returns without a launch).
"""
import ctypes as C

import pytest

BASE = 0x10000                 # fabricated, 16-byte aligned device address; operand k sits at BASE + k * 0x1000
ENTER_MESSAGES = ("CUDA driver unavailable", "cannot find the CUDA device", "null device pointer")
C_ = 64


def _lib():
    from xpretrain_b200 import _lib
    return _lib


def _m(ld=C_, group=0, group_stride=0):
    return _lib().XpRowMap(group=group, group_stride=group_stride, ld=ld, offsets=None)


def _ptrs(names, mis, shift):
    """{name: fabricated address}, `mis` moved by `shift` bytes."""
    return {n: BASE + k * 0x1000 + (shift if n == mis else 0) for k, n in enumerate(names)}


def _call(name, args):
    L = _lib()
    rc = getattr(L.lib(), name)(*args, None)
    return rc, (L.lib().xp_last_error().decode() if rc != 0 else "")


# case -> (entry point, the pointer operands it checks, builder of its arguments from {operand: address} and
# {operand: XpRowMap}, {operand with a row map: element size in bytes})
def _ln_fwd(x_dtype, y_dtype):
    def build(p, maps):
        return (p["x"], C.byref(maps["x"]), x_dtype, p["add"], C.byref(maps["add"]), p["sum_out"], C.byref(maps["sum_out"]),
                p["y"], C.byref(maps["y"]), y_dtype, p["gamma"], p["beta"], BASE, BASE, 0, C_, 1e-5)
    return build


def _ln_bwd(x_dtype):
    def build(p, maps):
        return (p["dy"], C.byref(maps["dy"]), p["x"], C.byref(maps["x"]), x_dtype, BASE, BASE, BASE, p["dres"],
                C.byref(maps["dres"]), p["dx"], C.byref(maps["dx"]), BASE, BASE, BASE if p["dres"] else 0, 0, C_)
    return build


def _cases():
    L = _lib()
    F32, BF16, F16 = L.DTYPE_F32, L.DTYPE_BF16, L.DTYPE_F16
    return {
        "xp_layernorm_add_fwd bf16": ("xp_layernorm_add_fwd", ["x", "add", "sum_out", "y", "gamma", "beta"],
                                      _ln_fwd(BF16, BF16), {"x": 2, "add": 2, "sum_out": 4, "y": 2}),
        "xp_layernorm_add_fwd fp32 x, fp16 y": ("xp_layernorm_add_fwd", ["x", "add", "sum_out", "y", "gamma", "beta"],
                                                _ln_fwd(F32, F16), {"x": 4, "add": 2, "sum_out": 4, "y": 2}),
        "xp_layernorm_add_fwd fp16": ("xp_layernorm_add_fwd", ["x", "add", "sum_out", "y", "gamma", "beta"],
                                      _ln_fwd(F16, F32), {"x": 2, "add": 2, "sum_out": 2, "y": 4}),
        "xp_layernorm_fwd": ("xp_layernorm_fwd", ["x", "y", "gamma", "beta"],
                             lambda p, m: (p["x"], C.byref(m["x"]), p["y"], C.byref(m["y"]), p["gamma"], p["beta"], BASE,
                                           BASE, 0, C_, 1e-5), {"x": 2, "y": 2}),
        "xp_layernorm_bwd bf16": ("xp_layernorm_bwd", ["dy", "x", "dres", "dx"], _ln_bwd(BF16),
                                  {"dy": 2, "x": 2, "dres": 2, "dx": 2}),
        "xp_layernorm_bwd fp32 x": ("xp_layernorm_bwd", ["dy", "x", "dres", "dx"], _ln_bwd(F32),
                                    {"dy": 2, "x": 4, "dres": 2, "dx": 2}),
        "xp_layernorm_wide_fwd": ("xp_layernorm_wide_fwd", ["x", "y"],
                                  lambda p, m: (p["x"], p["y"], BASE, BASE, BASE, BASE, 0, 2048, 1e-5), {}),
        "xp_layernorm_wide_bwd": ("xp_layernorm_wide_bwd", ["dy", "x", "dx"],
                                  lambda p, m: (p["dy"], p["x"], BASE, BASE, BASE, p["dx"], BASE, BASE, 0, 2048), {}),
        "xp_gather_rows_bf16": ("xp_gather_rows_bf16", ["src", "out"], lambda p, m: (p["src"], BASE, p["out"], 0, C_), {}),
        "xp_scatter_rows_bf16": ("xp_scatter_rows_bf16", ["in", "dst"], lambda p, m: (p["in"], BASE, p["dst"], 0, C_), {}),
        "xp_rowscale_bf16": ("xp_rowscale_bf16", ["x", "residual", "out"],
                             lambda p, m: (p["x"], BASE, p["residual"], p["out"], 0, C_), {}),
        "xp_colsum_bf16": ("xp_colsum_bf16", ["x"], lambda p, m: (p["x"], C_, BASE, 0, C_, 1.0), {}),
    }


CASES = ["xp_layernorm_add_fwd bf16", "xp_layernorm_add_fwd fp32 x, fp16 y", "xp_layernorm_add_fwd fp16",
         "xp_layernorm_fwd", "xp_layernorm_bwd bf16", "xp_layernorm_bwd fp32 x", "xp_layernorm_wide_fwd",
         "xp_layernorm_wide_bwd", "xp_gather_rows_bf16", "xp_scatter_rows_bf16", "xp_rowscale_bf16", "xp_colsum_bf16"]


def _assert_past_the_checks(what, rc, msg):
    assert rc == 0 or (any(m in msg for m in ENTER_MESSAGES) and "aligned" not in msg), \
        f"{what}: an aligned call must fail only at the CUDA driver, got {msg!r}"


@pytest.mark.parametrize("case", CASES)
def test_misaligned_operand_refused_before_the_driver(case):
    fn, names, build, elsize = _cases()[case]
    maps = {n: _m() for n in elsize}
    rc, msg = _call(fn, build(_ptrs(names, None, 0), maps))
    _assert_past_the_checks(f"{case}: all aligned", rc, msg)
    for name in names:
        for shift in (2, 4, 8):             # one bf16 / fp32 element, and half a vector
            rc, msg = _call(fn, build(_ptrs(names, name, shift), maps))
            assert rc != 0, f"{case}: {name} misaligned by {shift} bytes was accepted"
            assert f": {name} " in msg and "16-byte aligned" in msg, f"{case}: {name} +{shift}: message {msg!r}"
            assert not any(m in msg for m in ENTER_MESSAGES), msg


@pytest.mark.parametrize("case", [c for c in CASES if c.startswith("xp_layernorm_") and "wide" not in c])
def test_misaligned_row_map_refused_before_the_driver(case):
    """ld and group_stride times the element size must be multiples of 16 bytes; an explicit offsets table is device data
    and is not checked; group_stride is not used (and not checked) while group == 0, nor is the map of an optional
    operand passed as NULL."""
    fn, names, build, elsize = _cases()[case]
    p = _ptrs(names, None, 0)
    for name, es in elsize.items():
        step = 16 // es                                           # elements per 16 bytes; half of it is 8 bytes
        bad = {"ld": _m(ld=C_ + step // 2), "group_stride": _m(group=3, group_stride=5 * C_ + step // 2)}
        for field, rmap in bad.items():
            maps = {n: _m() for n in elsize}
            maps[name] = rmap
            rc, msg = _call(fn, build(p, maps))
            assert rc != 0, f"{case}: {name} row map with a misaligned {field} was accepted"
            assert f": {name} rows must be 16-byte aligned" in msg, f"{case}: {name} {field}: message {msg!r}"
        if name in ("add", "sum_out", "dres"):                   # an optional operand left NULL: its map is not read
            maps = {n: _m() for n in elsize}
            maps[name] = bad["ld"]
            q = dict(p, **{name: 0}, **({"sum_out": 0} if name == "add" else {}))
            rc, msg = _call(fn, build(q, maps))
            _assert_past_the_checks(f"{case}: NULL {name} with a misaligned map", rc, msg)
        ok = {"grouped": _m(group=3, group_stride=5 * C_ + step),
              "group_stride unused": _m(group=0, group_stride=1),
              "offsets": _lib().XpRowMap(group=0, group_stride=1, ld=1, offsets=BASE)}
        for label, rmap in ok.items():
            maps = {n: _m() for n in elsize}
            maps[name] = rmap
            rc, msg = _call(fn, build(p, maps))
            _assert_past_the_checks(f"{case}: {name} {label}", rc, msg)
