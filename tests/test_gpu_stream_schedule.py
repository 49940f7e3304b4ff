"""H100: the order of work across CUDA streams in CLIP-ViP's overlapped schedule, and the gradient-ready hook contract.

A CLIP-ViP step runs on three streams: the caller's ("main"); the text tower's forward and backward on a side stream under
the vision tower (`model.overlap_text_tower`); the vision backward's bias column sums on an auxiliary stream under its GEMMs
(`model.overlap_colsum`).  Every stream edge (`wait_stream`, `record_stream`, `_join_aux`) must hold whatever the timing.
At test sizes the text tower ends long before the vision tower, so a missing edge almost never shows by itself.

Harness.  Every kernel launch of the library goes through `ops._call` (test_boundary_cpu.py holds that to the header).
The `delay` fixture wraps it: before each launch on a stream whose role (main, side or aux) is delayed, it enqueues
`torch.cuda._sleep` on that stream, sized so that the stream falls behind by at least twice an undelayed step (one
counting pass gives the launches per role, one event-timed step the step time).  A sleep changes no result of correctly
ordered code; where an ordering edge is missing it turns a timing-dependent race into a reproducible wrong answer.  No
kernel, library source or model code changes.

Reading.  Every result is read in stream order on the caller's stream, with no synchronize in between: loss and features,
then a clone of every `.grad` right after `loss.backward()`.  Only then does the test synchronize and compare.  A
synchronize before the clones would wait for every stream, so a missing edge between a side stream and the caller's
stream could never show: the clones would read finished values whatever the model's own ordering.

Reference.  The same model, seed and inputs with `overlap_text_tower = overlap_colsum = False`, undelayed.  Loss and
features must have the same bits (the forward has no atomics, and GEMM results do not depend on the grid size); every
gradient must satisfy contract_harness.reordering_violations (max |g - g_ref| <= 1e-5 x scale).

Hook contract.  A recording `grad_ready_hook` clones each group's flat buffer at its hand-over, on the stream current then,
and clones every group again in `finish()` on the caller's stream.  Every snapshot must have the same bits as the group's
final contents; each backward hands over layers + 1 groups per tower that runs one, then calls `finish` once.

Negative controls plant a mistake with monkeypatch and show that the comparison reports it under the named delay.  A
planted mistake may only make floating-point data stale: those runs use a loss of plain elementwise kernels, so that memory
the caller's stream has freed but not yet finished with only ever holds float activations, and no kernel can read ids,
masks, offsets, pointer tables or workspace counters early.  No case loops waiting for a race.

`pytest -s` prints, per case and mode, the launches per stream, the per-launch sleep, the worst gradient ratio and the
number of hook groups.
"""
import collections

import pytest
import torch

from clipvip_cases import b16, l14, ragged_batch, vidclip
from contract_harness import GRAD_REL, reordering_violations, same_bits

pytestmark = pytest.mark.gpu

ROLES = ("main", "side", "aux")
MODES = {"none": (), "main": ("main",), "side": ("side",), "aux": ("aux",), "side+aux": ("side", "aux")}
REPORT = []


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda", 0)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if REPORT:
        print("\nstream schedule: launches main / side / aux | sleep per launch (us) | worst |g - g_ref| / scale | groups")
        for line in REPORT:
            print("  " + line)


@pytest.fixture(scope="module")
def cycles_per_ms(dev):
    """GPU clock cycles of torch.cuda._sleep per millisecond, from CUDA events around one sleep."""
    if not hasattr(torch.cuda, "_sleep"):
        pytest.fail("torch.cuda._sleep is missing: the schedule tests cannot delay a stream")
    torch.cuda._sleep(1000)
    n = 20_000_000
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    torch.cuda._sleep(n)
    e1.record()
    torch.cuda.synchronize()
    return n / e0.elapsed_time(e1)


class _Delay:
    """ops._call with a sleep in front of every launch on a delayed stream, counting launches per role."""

    def __init__(self, orig):
        self.orig, self.sleep, self.counts, self.main, self.model = orig, {}, collections.Counter(), None, None

    def role(self):
        h = torch.cuda.current_stream().cuda_stream
        if h == self.main:
            return "main"
        packs = self.model._packs if self.model is not None else {}
        for role, key in (("side", "overlap_text_tower"), ("aux", "overlap_colsum")):
            st = packs.get(key)
            if st is not None and st.cuda_stream == h:
                return role
        return "other"

    def __call__(self, name, *args):
        r = self.role()
        self.counts[r] += 1
        if self.sleep.get(r):
            torch.cuda._sleep(self.sleep[r])
        self.orig(name, *args)

    def run(self, model, step, sleep):
        """step() on the current stream as main, with `sleep` {role: cycles per launch}; synchronizes only after it."""
        self.main, self.model, self.sleep = torch.cuda.current_stream().cuda_stream, model, dict(sleep)
        self.counts.clear()
        try:
            res = step()
        finally:
            self.sleep = {}
        torch.cuda.synchronize()
        counts = dict(self.counts)
        assert counts.get("other", 0) == 0, f"{counts['other']} launches on a stream with no role"
        return res, counts


@pytest.fixture
def delay(monkeypatch, dev):
    from xpretrain_b200 import ops
    d = _Delay(ops._call)
    monkeypatch.setattr(ops, "_call", d)
    return d


def _calibrate(d, model, step, cpm):
    """Per-launch sleep (cycles) of each role, sized so that the role falls behind by twice an undelayed step."""
    _, counts = d.run(model, step, {})              # counting pass (also creates the streams and the weight copies)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    d.run(model, step, {})
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    return {r: int(2.0 * ms / counts[r] * cpm) for r in ROLES if counts.get(r)}, ms


class _Hook:
    """grad_ready_hook recording, per group, (flat, snapshot at hand-over, snapshot in finish())."""

    def __init__(self):
        self.log, self.groups, self.finish_streams = [], [], []

    def __call__(self, flat):
        self.log.append("group")
        self.groups.append([flat, flat.detach().clone(), None])

    def finish(self):
        self.log.append("finish")
        self.finish_streams.append(torch.cuda.current_stream().cuda_stream)
        for g in self.groups:
            if g[2] is None:
                g[2] = g[0].detach().clone()

    def violations(self, groups_per_call, calls, main):
        """groups_per_call: layers + 1 summed over the towers that run a backward.  With several backward calls, a group of
        an earlier call may be accumulated into afterwards (autograd adds the later call's gradient into the tensors it
        took as `.grad`): its snapshots are held to each other, the last call's to the final contents as well."""
        bad = []
        want = (["group"] * groups_per_call + ["finish"]) * calls if groups_per_call else []
        if self.log != want:
            bad.append(f"hook: hand-overs {self.log.count('group')}, finish calls {self.log.count('finish')}, order "
                       f"{''.join('g' if e == 'group' else 'F' for e in self.log)}; want {groups_per_call} groups then one "
                       f"finish, {calls} time(s)")
        if any(s != main for s in self.finish_streams):
            bad.append("hook: finish() ran on a stream other than the caller's")
        last = len(self.groups) - groups_per_call
        for i, (flat, at_hand, at_finish) in enumerate(self.groups):
            if at_finish is None or not same_bits(at_hand, at_finish):
                bad.append(f"hook group {i}: the hand-over snapshot differs from the one in finish()")
            elif i >= last and not same_bits(at_finish, flat):
                bad.append(f"hook group {i}: snapshots differ from the group's final contents")
        return bad


# ------------------------------------------------------------------------------------------------------ CLIP-ViP cases
def _model(dev, cfg=None, stream="fp32", per_frame=False):
    """B/16 at depth 2 unless `cfg` says otherwise; the ViP tower with its temporal table redrawn."""
    return vidclip(cfg or b16(2, 2), stream=stream, per_frame=per_frame, seed=0, temporal_init=not per_frame, dev=dev)


def _batch(dev, B=4, T=12, Lt=12, seed=1):
    video, ids, mask = ragged_batch(B, T, Lt, seed=seed, dev=dev)
    return {"video": video, "text_input_ids": ids, "text_input_mask": mask}


def _image_batch(dev, B=4, Lt=12, seed=2):
    b = _batch(dev, B, 1, Lt, seed)
    return {"image": b["video"], "caption_ids": b["text_input_ids"], "caption_masks": b["text_input_mask"]}


def _clip_step(model, batch, hook, train=True, loss_fn=None):
    """One step read in stream order on the current stream: ({name: output clone}, {name: .grad clone or None})."""
    from xpretrain_b200.optimization.loss import build_loss_func
    cm = model.clipmodel
    model.zero_grad(set_to_none=True)
    cm.grad_ready_hook = hook
    if not train:
        with torch.no_grad():
            out = model(**batch)
        return {"vis": out["vis_features"].clone(), "txt": out["text_features"].clone()}, {}
    out = model(**batch)
    feats = [out[k] for k in ("vis_features", "text_features", "img_features", "cap_features") if k in out]
    if loss_fn is not None:
        loss = loss_fn(*feats)
    elif len(feats) == 4:
        loss = build_loss_func({"loss_name": "NCELearnableTempLoss_vsc_fc"})(*feats, cm.logit_scale)
    else:
        loss = build_loss_func({"loss_name": "NCELearnableTempLoss"})(*feats, cm.logit_scale)
    loss.backward()
    outs = {"loss": loss.detach().clone()}
    outs.update({k: out[k].detach().clone() for k in ("vis_features", "text_features", "img_features", "cap_features")
                 if k in out})
    grads = {n: (p.grad.detach().clone() if p.grad is not None else None) for n, p in model.named_parameters()}
    return outs, grads


def _groups(model, train):
    """Hook groups per backward: layers + 1 for each tower that runs a backward."""
    cm = model.clipmodel
    if not train:
        return 0
    n = len(cm.vision_model.encoder.layers) + 1
    if any(p.requires_grad for p in cm.text_model.parameters()):
        n += len(cm.text_model.encoder.layers) + 1
    return n


def _set_overlap(model, on):
    model.clipmodel.overlap_text_tower = model.clipmodel.overlap_colsum = on


def _clip_run(d, model, batch, mode, sleep, overlap, train=True, loss_fn=None):
    """-> (outputs, grads, hook violations, launch counts)."""
    _set_overlap(model, overlap)
    hook = _Hook() if train else None
    calls = 2 if "image" in batch else 1
    try:
        (outs, grads), counts = d.run(model.clipmodel, lambda: _clip_step(model, batch, hook, train, loss_fn),
                                      {r: c for r, c in sleep.items() if r in MODES[mode]})
    finally:
        model.clipmodel.grad_ready_hook = None
    hook_bad = hook.violations(_groups(model, train), calls, d.main) if hook is not None else []
    return outs, grads, hook_bad, counts, (len(hook.groups) if hook is not None else 0)


def _record(case, mode, counts, sleep, cpm, worst, groups):
    line = (f"{case:22s} {mode:9s} {counts.get('main', 0):5d} / {counts.get('side', 0):4d} / {counts.get('aux', 0):3d} | "
            + " ".join(f"{r} {sleep[r] / cpm * 1e3:.1f}" for r in MODES[mode] if r in sleep).ljust(22)
            + f" | {worst[0]:.2e} ({worst[1]}) | {groups}")
    REPORT.append(line)
    print("  " + line)


def _clip_case(d, cpm, case, model, batch, modes, train=True):
    """The serial reference, then every mode of the overlapped schedule; asserts all rules, returns the reference."""
    ref_out, ref_g, hook_bad, _, _ = _clip_run(d, model, batch, "none", {}, False, train)
    assert not hook_bad, f"{case} serial: " + "; ".join(hook_bad)
    _set_overlap(model, True)
    sleep, _ = _calibrate(d, model.clipmodel, lambda: _clip_step(model, batch, _Hook() if train else None, train), cpm)
    model.clipmodel.grad_ready_hook = None
    failures = []
    for mode in modes:
        if any(r not in sleep for r in MODES[mode]):
            failures.append(f"{case} {mode}: no launches on {[r for r in MODES[mode] if r not in sleep]}")
            continue
        outs, grads, hook_bad, counts, groups = _clip_run(d, model, batch, mode, sleep, True, train)
        bad, worst = reordering_violations(ref_out, outs, ref_g, grads)
        _record(case, mode, counts, sleep, cpm, worst, groups)
        failures += [f"{case} {mode}: {b}" for b in bad + hook_bad]
    assert not failures, "\n".join(failures)
    return ref_out, ref_g


ALL = list(MODES)
CASES = {   # name: (model kwargs, batch kwargs, setup, modes, train)
    "vip_b16_fp32": ({}, {}, None, ALL, True),
    "vip_b16_eval": ({}, {}, "eval", ["none", "main", "side"], False),
    "checkpointing": ({}, {}, "ckpt", ALL, True),
    "fp16_stream": ({"stream": "fp16"}, {}, None, ALL, True),
    "bf16_stream": ({"stream": "bf16"}, {}, None, ALL, True),
    "frozen_text": ({}, {}, "frozen", ALL, True),
    "sm_reserve8": ({}, {}, "reserve", ALL, True),
    "per_frame_clip": ({"per_frame": True}, {}, None, ALL, True),
    "vit_l14_224_d1": ({"cfg": l14(224, 1, 1)}, {}, None, ALL, True),
    "image_caption": ({}, {}, "image", ALL, True),
}


@pytest.mark.parametrize("case", list(CASES))
def test_overlapped_schedule_matches_serial_under_forced_delays(dev, delay, cycles_per_ms, case):
    mkw, bkw, setup, modes, train = CASES[case]
    model = _model(dev, **mkw)
    batch = _batch(dev, **bkw)
    if setup == "eval":
        model.eval()
    elif setup == "ckpt":
        model.clipmodel.gradient_checkpointing_enable()
    elif setup == "frozen":
        model.freeze_text_encoder(freeze_text_proj=True)
    elif setup == "reserve":
        model.clipmodel.nccl_sm_reserve = 8
    elif setup == "image":
        batch.update(_image_batch(dev))
    _, ref_g = _clip_case(delay, cycles_per_ms, case, model, batch, modes, train)
    if setup == "frozen":
        assert all(g is None for n, g in ref_g.items() if ".text_model." in n or "text_projection" in n)


def test_bench_configuration_schedule(dev, delay, cycles_per_ms):
    """bench.py's workload, B = 64, T = 12, 12 + 12 layers.  Two serial runs also stay 5x inside the gradient bound of
    each other, so that the bound has room above the run-to-run reordering (measured 9.0e-7 and 1.02e-6 of the scale in two
    runs on an H100 80GB HBM3 at 700 W, about 10x inside; the overlapped-against-serial comparisons of the small cases
    reach 1.3e-6)."""
    model = _model(dev, b16(12, 12))
    batch = _batch(dev, B=64, T=12, Lt=32)
    ref_out, ref_g = _clip_case(delay, cycles_per_ms, "bench_b64_12+12", model, batch, ["none", "side", "aux"])
    outs, grads, hook_bad, _, _ = _clip_run(delay, model, batch, "none", {}, False)
    bad, worst = reordering_violations(ref_out, outs, ref_g, grads, rel=GRAD_REL / 5)
    print(f"  two serial runs of the bench configuration: worst gradient ratio {worst[0]:.2e} ({worst[1]})")
    assert not bad and not hook_bad, "\n".join(bad + hook_bad)


def test_weight_refresh_is_ordered_behind_the_side_stream(dev, delay, cycles_per_ms):
    """Two forwards with an in-place `p.data.mul_(0.5)` of every parameter on the caller's stream between them: the second
    forward must see the new weights and the first the old ones, whichever stream is behind."""
    model = _model(dev)
    batch = _batch(dev)
    params = list(model.parameters())
    start = [p.detach().clone() for p in params]

    def two_forwards():
        with torch.no_grad():
            for p, s in zip(params, start):
                p.data.copy_(s)
            first = model(**batch)
            first = {k + "_1": first[k].clone() for k in ("vis_features", "text_features")}
            for p in params:
                p.data.mul_(0.5)
            second = model(**batch)
        return dict(first, **{k + "_2": second[k].clone() for k in ("vis_features", "text_features")})

    _set_overlap(model, False)
    ref, _ = delay.run(model.clipmodel, two_forwards, {})
    _set_overlap(model, True)
    sleep, _ = _calibrate(delay, model.clipmodel, two_forwards, cycles_per_ms)
    failures = []
    for mode in ("none", "main", "side"):
        got, counts = delay.run(model.clipmodel, two_forwards, {r: c for r, c in sleep.items() if r in MODES[mode]})
        bad, _ = reordering_violations(ref, got, {}, {})
        _record("weight_refresh", mode, counts, sleep, cycles_per_ms, (0.0, None), 0)
        failures += [f"{mode}: {b}" for b in bad]
    assert not failures, "\n".join(failures)


# ---------------------------------------------------------------------------------------------- the caller's stream
def _on_user_stream(d, model, step, src, decoy, sleep, long_cycles):
    """step(*inputs) inside `with torch.cuda.stream(user)` with `user` delayed: the inputs reach `user` by copies issued
    after a long sleep, into buffers holding another valid batch (`decoy`), so that an early reader sees valid but wrong
    values."""
    dst = [t.clone() for t in decoy]
    user = torch.cuda.Stream()
    user.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(user):
        torch.cuda._sleep(long_cycles)
        for a, b in zip(dst, src):
            a.copy_(b)
        res, counts = d.run(model, lambda: step(*dst), {"main": sleep["main"]})
    torch.cuda.synchronize()
    return res, counts


def test_clip_vip_on_a_delayed_caller_stream(dev, delay, cycles_per_ms):
    model = _model(dev)
    batch, decoy = _batch(dev, seed=1), _batch(dev, seed=7)
    keys = list(batch)
    ref_out, ref_g, hook_bad, _, _ = _clip_run(delay, model, batch, "none", {}, False)
    assert not hook_bad, hook_bad
    _set_overlap(model, True)
    sleep, ms = _calibrate(delay, model.clipmodel, lambda: _clip_step(model, batch, None), cycles_per_ms)
    hook = _Hook()

    def step(*inputs):
        return _clip_step(model, dict(zip(keys, inputs)), hook)

    try:
        (outs, grads), counts = _on_user_stream(delay, model.clipmodel, step, [batch[k] for k in keys],
                                                [decoy[k] for k in keys], sleep, int(2 * ms * cycles_per_ms))
    finally:
        model.clipmodel.grad_ready_hook = None
    bad, worst = reordering_violations(ref_out, outs, ref_g, grads)
    bad += hook.violations(_groups(model, True), 1, delay.main)
    _record("vip_user_stream", "main", counts, sleep, cycles_per_ms, worst, len(hook.groups))
    assert not bad, "\n".join(bad)


def _encoder_check(d, cpm, case, model, x, decoy):
    """A TimeSformer or Swin-3D training step on a delayed caller's stream against the default-stream run."""
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():
        out0 = model(x)
    shape = (out0[0] if isinstance(out0, tuple) else out0).shape
    w = (torch.randn(shape, generator=g) / shape[1:].numel() ** 0.5).to(x.device)

    def step(inp):
        model.zero_grad(set_to_none=True)
        xin = inp.detach().requires_grad_(True)
        out = model(xin)
        out = out[0] if isinstance(out, tuple) else out
        (out.float() * w).sum().backward()
        grads = {n: (p.grad.detach().clone() if p.grad is not None else None) for n, p in model.named_parameters()}
        grads["input"] = xin.grad.detach().clone() if xin.grad is not None else None
        return {"out": out.detach().clone()}, grads

    (ref_out, ref_g), _ = d.run(None, lambda: step(x), {})
    sleep, ms = _calibrate(d, None, lambda: step(x), cpm)
    (outs, grads), counts = _on_user_stream(d, None, step, [x], [decoy], sleep, int(2 * ms * cpm))
    bad, worst = reordering_violations(ref_out, outs, ref_g, grads)
    _record(case, "main", counts, sleep, cpm, worst, 0)
    assert not bad, "\n".join(bad)


def test_timesformer_on_a_delayed_caller_stream(dev, delay, cycles_per_ms):
    from xpretrain_b200.modeling.timesformer import TimeSformer
    torch.manual_seed(0)
    model = TimeSformer(depth=2, num_frames=4, H=3, W=4, embed_dim=128, num_heads=2).to(dev).eval()
    g = torch.Generator().manual_seed(5)
    x, decoy = (torch.randn(3, 4, 128, 3, 4, generator=g).to(dev) for _ in range(2))
    _encoder_check(delay, cycles_per_ms, "timesformer_user", model, x, decoy)


def test_swin3d_on_a_delayed_caller_stream(dev, delay, cycles_per_ms):
    from oracle import swin3d_oracle as SO
    from xpretrain_b200.modeling.swin3d import SwinTransformer3D
    cfg = SO.Swin3DCfg(embed_dim=64, depths=(2, 2, 2), num_heads=(2, 4, 8), stages=(0, 1, 2), downsample_stages=(0, 1),
                       window_size=((2, 3, 5), (4, 3, 5), (8, 3, 5)))
    model = SwinTransformer3D(patch_size=list(cfg.patch_size), embed_dim=cfg.embed_dim, depths=list(cfg.depths),
                              num_heads=list(cfg.num_heads), stages=list(cfg.stages),
                              downsample_stages=list(cfg.downsample_stages),
                              window_size=[list(w) for w in cfg.window_size], patch_norm=cfg.patch_norm,
                              local_window=cfg.local_window, temporal_no_shifting=cfg.temporal_no_shifting)
    model.load_state_dict(SO.init_state_dict(cfg, seed=8), strict=True)
    model = model.to(dev).eval()
    x, decoy = (SO.synthetic_video(2, 4, 48, 80, cfg, seed=s).to(dev) for s in (9, 10))
    _encoder_check(delay, cycles_per_ms, "swin3d_user", model, x, decoy)


# --------------------------------------------------------------------------------------------------- negative controls
def _plant_join_aux_noop(monkeypatch, model):
    from xpretrain_b200.modeling import clip_vip
    monkeypatch.setattr(clip_vip, "_join_aux", lambda aux: None)


def _plant_colsum_without_wait(monkeypatch, model):
    from xpretrain_b200 import ops
    from xpretrain_b200.modeling import clip_vip

    def colsum(x, out, aux):
        if aux is None:
            ops.colsum(x, out)
            return
        with torch.cuda.stream(aux):          # no aux.wait_stream(current): may read x before it is written
            ops.colsum(x, out)
    monkeypatch.setattr(clip_vip, "_colsum", colsum)


def _plant_ignore_waits_on_side(monkeypatch, model):
    side = model.clipmodel._packs["overlap_text_tower"]
    orig = torch.cuda.Stream.wait_stream

    def wait_stream(self, stream):
        if stream.cuda_stream == side.cuda_stream:
            return None                       # drops main.wait_stream(side) in the forward and the backward
        return orig(self, stream)
    monkeypatch.setattr(torch.cuda.Stream, "wait_stream", wait_stream)


CONTROLS = {   # name: (planting function, the delay under which it must be caught)
    "join_aux_noop": (_plant_join_aux_noop, "aux"),
    "colsum_skips_wait": (_plant_colsum_without_wait, "main"),
    "main_ignores_side": (_plant_ignore_waits_on_side, "side"),
}


@pytest.mark.parametrize("name", list(CONTROLS))
def test_planted_ordering_mistake_is_caught(dev, delay, cycles_per_ms, monkeypatch, name):
    plant, mode = CONTROLS[name]
    model = _model(dev)
    batch = _batch(dev)
    g = torch.Generator().manual_seed(4)
    w = [(torch.randn(4, 512, generator=g) / 32).to(dev) for _ in range(2)]

    def loss_fn(vis, txt):      # elementwise kernels only (see the module docstring)
        return (vis * w[0]).sum() + (txt * w[1]).sum()

    ref_out, ref_g, hook_bad, _, _ = _clip_run(delay, model, batch, "none", {}, False, loss_fn=loss_fn)
    assert not hook_bad, hook_bad
    _set_overlap(model, True)
    sleep, _ = _calibrate(delay, model.clipmodel, lambda: _clip_step(model, batch, None, loss_fn=loss_fn), cycles_per_ms)
    plant(monkeypatch, model)
    found = {}
    for m in ("none", mode):
        outs, grads, hook_bad, counts, groups = _clip_run(delay, model, batch, m, sleep, True, loss_fn=loss_fn)
        bad, worst = reordering_violations(ref_out, outs, ref_g, grads)
        found[m] = bad + hook_bad
        _record(f"planted {name}", m, counts, sleep, cycles_per_ms, worst, groups)
    print(f"  planted {name}: {len(found['none'])} violations undelayed (not asserted), {len(found[mode])} under "
          f"{mode} delay, e.g. {found[mode][:2]}")
    assert found[mode], f"the planted mistake {name} went unnoticed under {mode} delay"
