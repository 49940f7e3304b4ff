"""H100: what the parameter layout (modeling/_weights.py) promises every model.  A weight written in place through `p.data`
(the reference AdamW's idiom, which autograd's version counter does not see) or by `load_state_dict` between two forwards
reaches the next forward, bit for bit as a freshly built model computes it; and TimeSformer evaluated under torch.no_grad()
keeps no activations."""
import json
from types import SimpleNamespace

import pytest
import torch

from clipvip_cases import b16, vidclip
from contract_harness import same_bits

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda", 0)


SWIN = dict(embed_dim=64, depths=[2, 2], num_heads=[2, 4], stages=[0, 1], downsample_stages=[0],
            window_size=[[2, 3, 5], [4, 3, 5]], patch_norm=True, local_window=4)


def _clip_vip(tmp):
    return vidclip(b16(1, 1))


def _clip_vip_inputs(dev, g):
    video = torch.randn(2, 2, 3, 224, 224, generator=g).to(dev)
    ids = torch.randint(1, 49407, (2, 16), generator=g).to(dev)
    return lambda m: tuple(m(video=video, text_input_ids=ids, text_input_mask=torch.ones_like(ids)).values())


def _tsf(tmp):
    from xpretrain_b200.modeling.timesformer import TimeSformer
    return TimeSformer(depth=2, num_frames=4, H=4, W=6, embed_dim=128, num_heads=2)


def _tsf_inputs(dev, g):
    x = torch.randn(2, 4, 128, 4, 6, generator=g).to(dev)
    return lambda m: (m(x),)


def _swin(tmp):
    from xpretrain_b200.modeling.swin3d import SwinTransformer3D
    return SwinTransformer3D(**SWIN)


def _swin_inputs(dev, g):
    video = torch.randn(2, 3, 4, 48, 80, generator=g).to(dev)
    return lambda m: m(video)[:1]


def _lfvila(tmp):
    from xpretrain_b200.modeling import LFVILA_Video_Classification
    path = tmp / "bert_config.json"
    path.write_text(json.dumps({"hidden_size": 128}))
    return LFVILA_Video_Classification(None, SimpleNamespace(VideoEncoder=SWIN, bert_config=str(path),
                                                             DATA=SimpleNamespace(classification_labels=5)))


def _lfvila_inputs(dev, g):
    video = torch.randn(2, 3, 4, 48, 80, generator=g).to(dev)
    labels = torch.tensor([1, 4], device=dev)
    return lambda m: tuple(v for k, v in m(video, labels).items() if k != "acc")


MODELS = {"clip_vip": (_clip_vip, _clip_vip_inputs), "timesformer": (_tsf, _tsf_inputs), "swin3d": (_swin, _swin_inputs),
          "lfvila_cls": (_lfvila, _lfvila_inputs)}


@pytest.mark.parametrize("name", sorted(MODELS))
def test_inplace_and_load_state_dict_updates_reach_the_next_forward(dev, tmp_path, name):
    from oracle import adamw_oracle as A
    build, inputs = MODELS[name]
    torch.manual_seed(0)
    model = build(tmp_path).to(dev).eval()
    run = inputs(dev, torch.Generator().manual_seed(1))
    sd0 = {k: v.clone() for k, v in model.state_dict().items()}
    with torch.no_grad():
        out0 = run(model)
    g = torch.Generator().manual_seed(2)
    versions = {n: p._version for n, p in model.named_parameters()}
    for n, p in model.named_parameters():                  # the reference AdamW step on p.data, from a seeded gradient
        grad = torch.randn(p.shape, generator=g).to(dev)
        A.adamw_step(p.data, grad, torch.zeros_like(p.data), torch.zeros_like(p.data), step=1, lr=1e-2, weight_decay=0.1)
    assert all(p._version == versions[n] for n, p in model.named_parameters())            # autograd did not notice
    with torch.no_grad():
        out1 = run(model)
    fresh = build(tmp_path)
    fresh.load_state_dict(model.state_dict())
    fresh = fresh.to(dev).eval()
    with torch.no_grad():
        want1 = run(fresh)
    assert all(same_bits(a, b) for a, b in zip(out1, want1)), name
    assert not same_bits(out1[0], out0[0]), name                                           # the step did move the output
    model.load_state_dict(sd0)
    with torch.no_grad():
        out2 = run(model)
    assert all(same_bits(a, b) for a, b in zip(out2, out0)), name


@pytest.mark.parametrize("attention_type", ["divided_space_time", "joint_space_time"])
def test_timesformer_evaluation_forward_keeps_no_activations(dev, attention_type):
    """Under torch.no_grad() the Function keeps nothing for a backward: 6 blocks of saved activations against one block's
    transients, the bar the CLIP-ViP test holds; the outputs are bitwise those of a forward with grad."""
    from xpretrain_b200.modeling.timesformer import TimeSformer
    torch.manual_seed(0)
    model = TimeSformer(depth=6, num_frames=8, H=16, W=16, embed_dim=256, num_heads=4,
                        attention_type=attention_type).to(dev).eval()
    x = torch.randn(2, 8, 256, 16, 16, generator=torch.Generator().manual_seed(3)).to(dev)
    with torch.no_grad():
        model(x)                                                      # the weight copies

    def peak(grad):
        torch.cuda.synchronize(); torch.cuda.empty_cache(); torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        with torch.set_grad_enabled(grad):
            out = model(x)
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base, out
    p_eval, ev = peak(False)
    p_train, tr = peak(True)
    print(f"{attention_type}: peak forward memory: eval {p_eval / 2**20:.1f} MiB, train {p_train / 2**20:.1f} MiB")
    assert tr.requires_grad and not ev.requires_grad
    assert p_eval < 0.5 * p_train
    assert same_bits(ev, tr.detach())
