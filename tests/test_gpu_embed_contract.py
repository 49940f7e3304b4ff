"""H100: the embedding kernels (embed.cu, tsf_embed.cu) against oracle/embed_ref.py, pinned on the CPU by
test_embed_reference_cpu.py.

  exact        patchify (every p and input dtype), the u8 transform, the ViP global rows, the non-interpolated table,
               text embeddings, the EOS index and both TimeSformer layout changes are bit-identical to the reference
  bound        the interpolated ViP table and the fp32-atomic backward sums are held element by element to embed_ref's
               derived bounds; the worst |err| / bound per kernel is printed at the end of the module
  taps         one-hot temporal rows read the kernel's interpolation weights back: a tap with more than ulp-level weight
               that the reference does not have fails; ulp-level drift at an integer source position is counted
  coverage     outputs live in NaN-filled buffers with guard regions: every element is written, pad columns are zero,
               xp_vip_embed_tables writes only the global rows of x, and nothing outside the outputs moves
  alignment    misaligned input views reach the kernels as aligned copies (checked on the host before any launch) and give
               the bits of the aligned call; misaligned outputs are refused before any launch
"""
import pytest
import torch

from contract_harness import Guarded, Report, same_bits, within
from oracle import embed_ref as E

pytestmark = pytest.mark.gpu

bf16, f32, f16, F64 = torch.bfloat16, torch.float32, torch.float16, torch.float64
REPORT = Report("embed: worst |err| / bound per kernel", width=40)
TAPS = {"checked": 0, "drifted": 0, "worst_drift": 0.0}


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda", 0)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    REPORT.print()
    if TAPS["checked"]:
        print(f"embed: {TAPS['checked']} interpolation taps checked; {TAPS['drifted']} moved to a neighbouring index with "
              f"ulp-level weight (largest {TAPS['worst_drift']:.3g})")


def _ops():
    from xpretrain_b200 import ops
    return ops


def _lib():
    from xpretrain_b200 import _lib
    return _lib


def _launches():
    return int(_ops().launch_count())


# ============================================================================================== patchify
# (frames, H, W) per patch size: non-square, frames 1 ... 37; p = 4 and 8 are Swin-3D's PatchEmbed3D launches
SHAPES = {4: [(1, 8, 12), (37, 4, 8), (16, 64, 96)], 8: [(16, 224, 224)], 14: [(1, 14, 28), (3, 28, 42), (37, 14, 14)],
          16: [(1, 32, 48), (5, 16, 16), (37, 48, 32)], 32: [(2, 64, 32), (37, 32, 32)]}
CASES = [(p, s) for p, ss in SHAPES.items() for s in ss]


def _video(dev, frames, H, W, dtype, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    if dtype == torch.uint8:
        return torch.randint(0, 256, (frames, H, W, 3), generator=g, device=dev, dtype=torch.uint8)
    x = torch.randn(frames, 3, H, W, generator=g, device=dev) * 3
    x[0, 0, 0, :2] = torch.tensor([65504.0 if dtype == f16 else 1e30, -0.0])          # large and signed-zero inputs
    return x.to(dtype)


@pytest.mark.parametrize("dtype", [f32, bf16, f16, torch.uint8], ids=["f32", "bf16", "f16", "u8"])
@pytest.mark.parametrize("p,shape", CASES, ids=[f"p{p}-{f}x{h}x{w}" for p, (f, h, w) in CASES])
def test_patchify_is_exact_and_writes_exactly_the_patch_matrix(dev, p, shape, dtype):
    ops = _ops()
    frames, H, W = shape
    video = _video(dev, frames, H, W, dtype, seed=frames * 131 + p)
    rows, ld = frames * (H // p) * (W // p), E.patch_pitch(p)
    out = Guarded(dev, (rows, ld), bf16)
    if dtype == torch.uint8:
        ops.vip_patchify_u8(video, out.t, p)
        want = E.patchify_u8_ref(video, p, ops.CLIP_MEAN, ops.CLIP_STD)
    else:
        ops.vip_patchify(video, out.t, p)
        want = E.patchify_ref(video, p)
    got = out.written(f"patchify p={p} {dtype}")
    assert same_bits(got, want), f"p={p} {dtype}: {int((got.view(torch.int16) != want.view(torch.int16)).sum())} elements differ"
    assert torch.all(got[:, 3 * p * p:].view(torch.int16) == 0), "pad columns must be +0"


# ============================================================================================== ViP tables
def _tables(dev, C, M, Tsz, L, seed, temporal="random"):
    g = torch.Generator(device=dev).manual_seed(seed)
    pos = torch.randn(L + 1, C, generator=g, device=dev)
    if temporal == "onehot":
        tmp = torch.eye(Tsz, C, device=dev)
        pos.zero_()
    elif temporal == "random":        # rows with large, distinct offsets: a wrong tap cannot hide inside the bound
        tmp = torch.randn(Tsz, C, generator=g, device=dev) + 64.0 * torch.arange(Tsz, device=dev, dtype=f32)[:, None]
    else:
        tmp = None
    cls = torch.randn(C, generator=g, device=dev)
    added = torch.randn(max(M - 1, 1), C, generator=g, device=dev)
    return pos, tmp, cls, added


def _run_tables(dev, B, T, L, M, C, Tsz, pos, tmp, cls, added):
    ops = _ops()
    S = M + T * L
    table = Guarded(dev, (T * L, C), bf16)
    x0 = Guarded(dev, (B * S, C), bf16)
    ops.vip_embed_tables(pos, tmp, cls, added if M > 1 else None, table.t, x0.t, B, T, L, M, C, Tsz)
    tab = table.written("table")
    x0.guards("x0")
    x = x0.t.view(B, S, C)
    assert torch.isnan(x[:, M:]).all(), "xp_vip_embed_tables wrote into the patch rows of x"
    return tab, x[:, :M]


TABLE_CASES = ([(12, T, 4, 768) for T in range(1, 33)] + [(1, 1, 4, 512), (1, 5, 4, 512)]
               + [(12, T, M, C) for T in (5, 12, 16) for M in (1, 4, 8) for C in (512, 768, 1024, 200)])


@pytest.mark.parametrize("Tsz,T,M,C", TABLE_CASES)
def test_vip_tables_within_bound_and_global_rows_exact(dev, Tsz, T, M, C):
    B, L = 3, 7
    pos, tmp, cls, added = _tables(dev, C, M, Tsz, L, seed=T * 97 + M * 13 + C)
    tab, glob = _run_tables(dev, B, T, L, M, C, Tsz, pos, tmp, cls, added)
    exact, bound, t32, want_glob = E.vip_tables_ref(pos, tmp, cls, added, B, T, L, M, Tsz)
    assert same_bits(glob, want_glob), "global rows differ from bf16(fp32(embedding + pos[0]))"
    if t32 is not None:
        assert same_bits(tab, t32), "non-interpolated table differs from bf16(fp32(temporal + pos))"
    else:
        within(REPORT, "vip_embed_tables (interpolated)", tab, exact, bound)


@pytest.mark.parametrize("T", [1, 4, 12, 32])
def test_vip_tables_null_temporal_is_the_position_table(dev, T):
    B, L, M, C = 2, 5, 4, 256
    pos, _, cls, added = _tables(dev, C, M, 12, L, seed=T, temporal=None)
    tab, glob = _run_tables(dev, B, T, L, M, C, 12, pos, None, cls, added)
    assert same_bits(tab, pos[1:1 + L].to(bf16).repeat(T, 1))


@pytest.mark.parametrize("Tsz,T", [(12, T) for T in range(1, 33)] + [(1, 1), (1, 6), (5, 3)])
def test_interpolation_taps_are_exact(dev, Tsz, T):
    """temporal = identity rows and pos = 0: table[t*L, k] is the kernel's weight of temporal row k for frame t."""
    B, L, M, C = 1, 2, 1, 64
    pos, tmp, cls, added = _tables(dev, C, M, Tsz, L, seed=1, temporal="onehot")
    tab, _ = _run_tables(dev, B, T, L, M, C, Tsz, pos, tmp, cls, added)
    got = tab.view(T, L, C)[:, 0, :Tsz].to(F64).cpu()
    assert torch.equal(tab.view(T, L, C)[:, 1], tab.view(T, L, C)[:, 0]), "rows of one frame differ"
    assert torch.all(tab.view(T, L, C)[:, :, Tsz:].float() == 0)
    Wm = E.tap_matrix(Tsz, T)
    dw = E.weight_error(Tsz, T)
    tol = dw + 2 * E.U + 0.5 * E.ulp_bf16(Wm + dw)            # the weight's own error, 1 - w1 rounding, the bf16 readout
    err = (got - Wm).abs()
    assert torch.all(err <= tol), f"T={T}: a tap weight is off by {float(err.max()):.3g} (allowed {float(tol.max()):.3g})"
    drift = (got != 0) != (Wm != 0)
    TAPS["checked"] += T
    if bool(drift.any()):
        TAPS["drifted"] += int(drift.any(dim=1).sum())
        TAPS["worst_drift"] = max(TAPS["worst_drift"], float(torch.maximum(got, Wm)[drift].max()))


# ============================================================================================== ViP backward
def _bwd_case(dev, B, T, L, M, C, Tsz, seed, with_temporal=True, with_cls=True, with_added=True):
    ops = _ops()
    g = torch.Generator(device=dev).manual_seed(seed)
    d_patch = (torch.randn(B * T * L, C, generator=g, device=dev)).to(bf16)
    d_glob = (torch.randn(B * M, C, generator=g, device=dev)).to(bf16)
    init = {"pos": torch.randn(L + 1, C, generator=g, device=dev), "temporal": torch.randn(Tsz, C, generator=g, device=dev),
            "cls": torch.randn(C, generator=g, device=dev), "added": torch.randn(max(M - 1, 1), C, generator=g, device=dev)}
    use = {"pos": True, "temporal": with_temporal, "cls": with_cls, "added": with_added and M > 1}
    outs = {k: Guarded(dev, tuple(v.shape), f32, init=v) for k, v in init.items()}
    ops.vip_embed_bwd(d_patch, d_glob, outs["pos"].t, outs["temporal"].t if use["temporal"] else None,
                      outs["cls"].t if use["cls"] else None, outs["added"].t if use["added"] else None,
                      B, T, L, M, C, Tsz)
    ref = E.vip_bwd_ref(d_patch, d_glob, {k: (init[k] if use[k] else None) for k in init} | {"pos": init["pos"],
                        "cls": init["cls"]}, B, T, L, M, Tsz)
    for k, o in outs.items():
        got = o.written(f"vip_embed_bwd d_{k}")
        if not use[k]:
            assert same_bits(got, init[k]), f"d_{k} was not requested but changed"
            continue
        within(REPORT, f"vip_embed_bwd d_{k}", got, *ref[k])


@pytest.mark.parametrize("Tsz,T,M,C", [(12, 12, 4, 768), (12, 5, 8, 512), (12, 32, 4, 1024), (12, 16, 1, 200),
                                       (12, 1, 4, 768), (1, 4, 4, 512), (12, 13, 8, 1024)])
def test_vip_embed_bwd_accumulates_within_bound(dev, Tsz, T, M, C):
    _bwd_case(dev, 4, T, 7, M, C, Tsz, seed=T * 5 + M)


@pytest.mark.parametrize("which", ["temporal", "cls", "added", "all"])
def test_vip_embed_bwd_optional_destinations(dev, which):
    """NULL d_temporal / d_cls / d_added: that gradient is not wanted; M = 1 needs no added_cls at all."""
    kw = {"with_temporal": which not in ("temporal", "all"), "with_cls": which not in ("cls", "all"),
          "with_added": which not in ("added", "all")}
    _bwd_case(dev, 3, 6, 5, 4, 256, 12, seed=3, **kw)
    _bwd_case(dev, 3, 6, 5, 1, 256, 12, seed=4, **kw)


@pytest.mark.parametrize("C", [12, 1032])
def test_vip_embed_bwd_refuses_bad_widths_before_any_launch(dev, C):
    ops = _ops()
    B, T, L, M = 2, 3, 4, 2
    d_patch = torch.zeros(B * T * L, C, dtype=bf16, device=dev)
    d_glob = torch.zeros(B * M, C, dtype=bf16, device=dev)
    d_pos = torch.zeros(L + 1, C, device=dev)
    n0 = _launches()
    with pytest.raises(_lib().XpError):
        ops.vip_embed_bwd(d_patch, d_glob, d_pos, None, None, None, B, T, L, M, C, 12)
    assert _launches() == n0


# ============================================================================================== text
TEXT = [(1, 1, 512), (3, 5, 200), (2, 33, 512), (4, 77, 512), (2, 77, 1028), (1, 77, 4)]


@pytest.mark.parametrize("B,Lt,C", TEXT)
@pytest.mark.parametrize("kind", ["random", "padding", "out_of_range"])
def test_text_embeddings(dev, B, Lt, C, kind):
    ops = _ops()
    vocab = 1000
    g = torch.Generator(device=dev).manual_seed(B * Lt + C)
    tok = torch.randn(vocab, C, generator=g, device=dev)
    pos = torch.randn(Lt, C, generator=g, device=dev)
    ids = torch.randint(0, vocab, (B, Lt), generator=g, device=dev)
    ids.view(-1)[0] = 0
    ids.view(-1)[-1] = vocab - 1
    if kind == "padding":                      # one id in every row: the most atomic contention in the backward
        ids.fill_(vocab - 1)
    if kind == "out_of_range":
        ids.view(-1)[-1] = vocab
        ids.view(-1)[0] = -3
    x = Guarded(dev, (B * Lt, C), bf16)
    err = torch.zeros(1, dtype=torch.int32, device=dev)
    ops.text_embed_fwd(ids, tok, pos, x.t, Lt, err)
    want, flag = E.text_fwd_ref(ids, tok, pos, Lt)
    assert same_bits(x.written("text_embed_fwd"), want)
    assert int(err.item()) == flag == (1 if kind == "out_of_range" else 0)
    dx = torch.randn(B * Lt, C, generator=g, device=dev).to(bf16)
    t0, p0 = torch.randn(vocab, C, generator=g, device=dev), torch.randn(Lt, C, generator=g, device=dev)
    d_tok, d_pos = Guarded(dev, (vocab, C), f32, init=t0), Guarded(dev, (Lt, C), f32, init=p0)
    ops.text_embed_bwd(ids, dx, d_tok.t, d_pos.t, Lt, C, vocab)
    ref = E.text_bwd_ref(ids, dx, t0, p0, Lt)
    within(REPORT, "text_embed_bwd d_tok", d_tok.written("d_tok"), *ref["tok"])
    within(REPORT, "text_embed_bwd d_pos", d_pos.written("d_pos"), *ref["pos"])


# ============================================================================================== EOS
@pytest.mark.parametrize("B", [1, 7, 1024])
@pytest.mark.parametrize("Lt", [1, 31, 32, 33, 77])
def test_eos_first_maximum_exact(dev, B, Lt):
    ops = _ops()
    g = torch.Generator(device=dev).manual_seed(B * 100 + Lt)
    ids = torch.randint(-50, 6, (B, Lt), generator=g, device=dev)         # few values: ties within and across lanes
    ids[0] = -9                                                            # all tied, all negative
    if B > 1:
        ids[1] = torch.randint(-9, -1, (Lt,), generator=g, device=dev)     # negative maximum
    if B > 2 and Lt > 33:
        ids[2].fill_(0)
        ids[2, 33] = ids[2, 1] = 7                                         # a tie inside lane 1 (its first and second pass)
    off = Guarded(dev, (B,), torch.int64)
    idx = Guarded(dev, (B,), torch.int32)
    ops.eos_offsets(ids, off.t, idx.t, 512)
    want_off, want_idx = E.eos_ref(ids, 512)
    off.guards("offsets")
    idx.guards("index")
    assert torch.equal(idx.t, want_idx) and torch.equal(off.t, want_off)
    assert torch.equal(want_idx.long(), ids.argmax(dim=1))


# ============================================================================================== TimeSformer tokens
TSF = [(hw, c) for hw in (1, 49, 63, 196) for c in (1, 31, 33, 768)]


@pytest.mark.parametrize("dtype", [f32, bf16, f16], ids=["f32", "bf16", "f16"])
@pytest.mark.parametrize("HW,C", TSF)
def test_tsf_tokens_and_untokenize_exact(dev, HW, C, dtype):
    B, T = 2, 3
    for tables in ("both", "pos", "time", "none"):
        _tsf_roundtrip(dev, B, T, C, HW, dtype, tables, seed=HW * 7 + C)


def _tsf_roundtrip(dev, B, T, C, HW, dtype, tables, seed):
    ops = _ops()
    g = torch.Generator(device=dev).manual_seed(seed)
    x = (torch.randn(B, T, C, HW, generator=g, device=dev) * 2).to(dtype)
    pos = torch.randn(HW, C, generator=g, device=dev) if tables in ("both", "pos") else None
    time = torch.randn(T, C, generator=g, device=dev) if tables in ("both", "time") else None
    tok = Guarded(dev, (B * HW * T, C), bf16)
    ops.tsf_embed_fwd(x, pos, time, tok.t, B, T, C, HW)
    got = tok.written(f"tsf tokens {tables}")
    assert same_bits(got, E.tsf_tokens_ref(x, pos, time)), f"tokens ({tables}) differ"
    back = Guarded(dev, (B, T, C, HW), dtype)
    ops.tsf_untokenize(got, back.t, B, T, C, HW)
    assert same_bits(back.written("untokenize"), E.tsf_untokenize_ref(got, B, T, C, HW, dtype))


@pytest.mark.parametrize("B,T", [(1, 1), (1, 65535), (65535, 1), (5, 13107)])
def test_tsf_grid_limit(dev, B, T):
    _tsf_roundtrip(dev, B, T, 1, 1, f32, "both", seed=B + T)


@pytest.mark.parametrize("B,T", [(1, 65536), (2, 32768)])
def test_tsf_refuses_65536_sequences_before_any_launch(dev, B, T):
    ops = _ops()
    x = torch.zeros(B, T, 1, 1, device=dev)
    tok = torch.empty(B * T, 1, dtype=bf16, device=dev)
    n0 = _launches()
    with pytest.raises(_lib().XpError):
        ops.tsf_embed_fwd(x, None, None, tok, B, T, 1, 1)
    with pytest.raises(_lib().XpError):
        ops.tsf_untokenize(tok, x, B, T, 1, 1)
    assert _launches() == n0


# ============================================================================================== alignment
def _misaligned(t, offset_elems=1):
    """A contiguous copy of t whose data pointer is offset_elems elements past a 64-byte boundary."""
    buf = torch.empty(t.numel() + offset_elems, dtype=t.dtype, device=t.device)
    view = buf[offset_elems:].view(t.shape)
    view.copy_(t)
    return view


def _checked(monkeypatch, name, arg_align):
    """Wrap the C entry point `name` so that, on the host and before the call, every (argument index, alignment) of
    arg_align is asserted; a misaligned pointer never reaches the library."""
    h = _lib().lib()
    orig = getattr(h, name)
    calls = []

    def wrapper(*args):
        for i, a in arg_align:
            assert args[i] is None or args[i] % a == 0, f"{name}: argument {i} is misaligned ({args[i] % a} mod {a})"
        calls.append(args)
        return orig(*args)
    monkeypatch.setattr(h, name, wrapper)
    return calls


@pytest.mark.parametrize("p", [14, 16])
@pytest.mark.parametrize("dtype", [f32, bf16, f16], ids=["f32", "bf16", "f16"])
def test_patchify_copies_a_misaligned_video(dev, monkeypatch, dtype, p):
    ops = _ops()
    video = _video(dev, 3, 2 * p, 3 * p, dtype, seed=p)
    rows, ld = 3 * 6, E.patch_pitch(p)
    want = torch.empty(rows, ld, dtype=bf16, device=dev)
    ops.vip_patchify(video, want, p)
    calls = _checked(monkeypatch, "xp_vip_patchify", [(0, 16), (2, 16)])
    got = Guarded(dev, (rows, ld), bf16)
    mis = _misaligned(video)
    assert mis.is_contiguous() and mis.data_ptr() % 16 != 0
    ops.vip_patchify(mis, got.t, p)
    assert len(calls) == 1 and same_bits(got.written("patchify (misaligned video)"), want)


def test_patchify_u8_copies_misaligned_frames(dev, monkeypatch):
    ops = _ops()
    frames = _video(dev, 2, 32, 48, torch.uint8, seed=9)
    want = torch.empty(2 * 6, 768, dtype=bf16, device=dev)
    ops.vip_patchify_u8(frames, want, 16)
    calls = _checked(monkeypatch, "xp_vip_patchify_u8", [(0, 8), (1, 16)])
    got = torch.empty_like(want)
    ops.vip_patchify_u8(_misaligned(frames, 3), got, 16)
    assert len(calls) == 1 and same_bits(got, want)


@pytest.mark.parametrize("entry", ["xp_vip_patchify", "xp_vip_patchify_u8"])
def test_patchify_refuses_a_misaligned_output(dev, monkeypatch, entry):
    ops = _ops()
    u8 = entry.endswith("u8")
    video = _video(dev, 2, 32, 32, torch.uint8 if u8 else f32, seed=2)
    calls = _checked(monkeypatch, entry, [(1 if u8 else 2, 16)])
    out = _misaligned(torch.zeros(2 * 4, 768, dtype=bf16, device=dev), 4)      # 8 bytes past a boundary
    n0 = _launches()
    with pytest.raises(_lib().XpError):
        (ops.vip_patchify_u8 if u8 else ops.vip_patchify)(video, out, 16)
    assert not calls and _launches() == n0


def test_text_embed_copies_misaligned_tables_and_refuses_a_misaligned_output(dev, monkeypatch):
    ops = _ops()
    vocab, C, Lt = 300, 512, 77
    g = torch.Generator(device=dev).manual_seed(0)
    tok = torch.randn(vocab, C, generator=g, device=dev)
    pos = torch.randn(Lt, C, generator=g, device=dev)
    ids = torch.randint(0, vocab, (2, Lt), generator=g, device=dev)
    err = torch.zeros(1, dtype=torch.int32, device=dev)
    want = torch.empty(2 * Lt, C, dtype=bf16, device=dev)
    ops.text_embed_fwd(ids, tok, pos, want, Lt, err)
    calls = _checked(monkeypatch, "xp_text_embed_fwd", [(1, 16), (2, 16), (3, 8)])
    got = torch.empty_like(want)
    ops.text_embed_fwd(ids, _misaligned(tok), _misaligned(pos, 2), got, Lt, err)
    assert len(calls) == 1 and same_bits(got, want)
    n0 = _launches()
    with pytest.raises(_lib().XpError):
        ops.text_embed_fwd(ids, tok, pos, _misaligned(want, 1), Lt, err)
    assert len(calls) == 1 and _launches() == n0


def test_vip_embed_bwd_copies_misaligned_gradients(dev, monkeypatch):
    ops = _ops()
    B, T, L, M, C = 2, 4, 5, 4, 256
    g = torch.Generator(device=dev).manual_seed(1)
    d_patch = torch.randn(B * T * L, C, generator=g, device=dev).to(bf16)
    d_glob = torch.randn(B * M, C, generator=g, device=dev).to(bf16)
    calls = _checked(monkeypatch, "xp_vip_embed_bwd", [(0, 16), (1, 16)])
    d_pos = torch.zeros(L + 1, C, device=dev)
    ops.vip_embed_bwd(_misaligned(d_patch, 3), _misaligned(d_glob, 1), d_pos, None, None, None, B, T, L, M, C, 12)
    ref = E.vip_bwd_ref(d_patch, d_glob, {"pos": torch.zeros_like(d_pos), "cls": torch.zeros(C, device=dev)}, B, T, L, M, 12)
    assert len(calls) == 1
    within(REPORT, "vip_embed_bwd d_pos (misaligned input)", d_pos, *ref["pos"])
