"""What the measurement tools share: the card record every printed line carries, the two CUDA-event timing methods, peak
memory, profiler kernel time, and the CLIP-ViP training step.

Two timing methods, for two questions: `window_ms` is the mean over a window of back-to-back calls (a step time, as a
training loop sees it); `median_ms` is the median of single calls, each after an L2 flush (a kernel's cold-cache time).
"""
import json
import subprocess
import sys
from types import SimpleNamespace

import torch

from oracle import clipvip_oracle as O
from xpretrain_b200.modeling import VidCLIP
from xpretrain_b200.optimization.loss import gather_nce_loss

NO_GPU = "this tool measures on a GPU, and torch.cuda.is_available() is False"
GIB = 2 ** 30


def require_gpu():
    if not torch.cuda.is_available():
        sys.exit(NO_GPU)


def card(index=0):
    """The card's name, power limit and SM clocks (maximum and current), read now; a field that cannot be read is None."""
    rec = {"name": None, "power_limit_w": None, "max_sm_mhz": None, "sm_mhz": None}
    try:
        rec["name"] = torch.cuda.get_device_name(index)
    except Exception:  # noqa: BLE001 - no device, no driver: the record says so with None
        pass
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader,nounits",
                            "-i", str(index)], capture_output=True, text=True, timeout=30)
    except (OSError, subprocess.SubprocessError):
        return rec
    lines = q.stdout.strip().splitlines() if q.returncode == 0 else []
    for (key, kind), text in zip((("power_limit_w", float), ("max_sm_mhz", int), ("sm_mhz", int)),
                                 lines[0].split(",") if lines else []):
        try:
            rec[key] = kind(float(text))
        except ValueError:          # "[N/A]", "[Not Supported]"
            pass
    return rec


def emit(record):
    """Print `record` as one JSON line with the card read in the same call, and return the line."""
    line = json.dumps({**record, "card": card()})
    print(line, flush=True)
    return line


def window_ms(fn, steps, warmup):
    """Mean ms per call of `steps` back-to-back calls after `warmup` calls: one event pair around the window."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def median_ms(fn, iters, warmup, flush=None):
    """Median ms of `iters` single calls after `warmup` calls, one event pair each, `flush` zeroed before each call."""
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        if flush is not None:
            flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


def peak_gib(fn):
    """(fn's result, the peak memory allocated while it ran, in GiB; tensors alive at the call count)."""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    res = fn()
    torch.cuda.synchronize()
    return res, torch.cuda.max_memory_allocated() / GIB


def profiled_kernel_ms(fn, names=()):
    """(total, named) device ms of the CUDA kernels of one call of `fn` under torch.profiler, after one untimed call;
    `named` sums the kernels whose name contains one of `names`."""
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    evs = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    total = sum(e.device_time for e in evs) / 1e3
    named = sum(e.device_time for e in evs if any(k in e.name for k in names)) / 1e3
    return total, named


def clip_model(dev, config_name, vision_type="ViP", seed_temporal=False):
    """VidCLIP from `config_name`'s widths with seed-0 weights; `seed_temporal` draws the temporal embedding from
    N(0, 0.02) instead of its zero initialisation."""
    add = SimpleNamespace(type=vision_type, temporal_size=12, if_use_temporal_embed=1, logit_scale_init_value=4.60,
                          add_cls_num=3)
    torch.manual_seed(0)
    model = VidCLIP(SimpleNamespace(clip_config=config_name, clip_weights="", clip_vision_additional_config=add))
    if seed_temporal:
        with torch.no_grad():
            model.clipmodel.vision_model.embeddings.temporal_embedding.normal_(0, 0.02)
    return model.to(dev)


def clip_batch(dev, B, T, size, Lt):
    """(video [B, T, 3, size, size], text ids [B, Lt] ending in the end-of-text token, all-ones mask), seeded."""
    g = torch.Generator().manual_seed(1234)
    video = torch.randn(B, T, 3, size, size, generator=g)
    ids = torch.randint(1, 49406, (B, Lt), generator=g)
    ids[:, -1] = 49407
    return video.to(dev), ids.to(dev), torch.ones(B, Lt, dtype=torch.long, device=dev)


def clip_train_step(model, batch):
    """Zero the gradients, forward, fused gather_nce_loss, backward.  Returns (loss, the model's outputs)."""
    for p in model.parameters():
        p.grad = None
    out = model(video=batch[0], text_input_ids=batch[1], text_input_mask=batch[2])
    loss = gather_nce_loss(out["vis_features"], out["text_features"], model.clipmodel.logit_scale)
    loss.backward()
    return loss, out


def eager_oracle_step(model, batch, forward):
    """A step function: the oracle's `forward(state_dict, video, ids, mask)` + InfoNCE + backward in PyTorch eager under
    bf16 autocast, on fp32 copies of `model`'s weights (the reference's mixed precision)."""
    sd = {k: (v.detach().clone().requires_grad_(True) if v.is_floating_point() else v)
          for k, v in model.clipmodel.state_dict().items()}

    def step():
        for v in sd.values():
            if v.is_floating_point():
                v.grad = None
        with torch.autocast("cuda", dtype=torch.bfloat16):
            o = forward(sd, *batch)
            loss = O.nce_learnable_temp_loss(o["vis_features"].float(), o["text_features"].float(), sd["logit_scale"].float())
        loss.backward()
    return step
