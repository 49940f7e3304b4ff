"""H100: the TimeSformer token kernels (tsf_embed.cu) at the settings the model runs them, element by element.

  forward      xp_tsf_embed_fwd from f32 (the module's input), bf16 or f16 x, with both tables, the position table only,
               or none (the tokenizer of the output gradient): bit-exact against bf16((x + pos) + time) in fp32, the
               kernel's order (oracle/embed_ref.tsf_tokens_ref)
  untokenize   xp_tsf_untokenize into f32, bf16 and f16: bit-exact against the bf16 -> dtype cast; for f16 that is torch's
               cast, overflow to inf and subnormals included
  shapes       C in {1, 31, 33, 768, 1024}, H*W in {1, 31, 49, 160, 784}, T in {1, 7, 8}, B up to 4: the 32 x 32 tiles are
               ragged in C and H*W
  coverage     every output lives in a NaN-filled buffer with guard bytes: every element written, nothing outside it
The B*T grid limit (65535 runs, 65536 refused before any launch) is tested in test_gpu_embed_contract.py.
"""
import pytest
import torch

from contract_harness import Guarded, same_bits
from oracle import embed_ref as E

pytestmark = pytest.mark.gpu

bf16, f32, f16 = torch.bfloat16, torch.float32, torch.float16
CS = (1, 31, 33, 768, 1024)
HWS = (1, 31, 49, 160, 784)
BT = ((4, 1), (1, 7), (2, 8))


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda", 0)


def _ops():
    from xpretrain_b200 import ops
    return ops


def _tokens(dev, x, pos, time, B, T, C, HW):
    tok = Guarded(dev, (B * HW * T, C), bf16)
    _ops().tsf_embed_fwd(x, pos, time, tok.t, B, T, C, HW)
    return tok.written(f"tokens B{B} T{T} C{C} HW{HW} {x.dtype}")


@pytest.mark.parametrize("B,T", BT, ids=[f"B{b}T{t}" for b, t in BT])
@pytest.mark.parametrize("HW", HWS)
@pytest.mark.parametrize("C", CS)
def test_tokens_and_untokenize_are_exact(dev, C, HW, B, T):
    g = torch.Generator(device=dev).manual_seed(C * 1009 + HW * 31 + T)
    x32 = torch.randn(B, T, C, HW, generator=g, device=dev) * 3
    pos = torch.randn(HW, C, generator=g, device=dev)
    time = torch.randn(T, C, generator=g, device=dev)
    for dtype in (f32, bf16, f16):
        x = x32.to(dtype)
        for tables in ((pos, time), (pos, None), (None, None)):
            got = _tokens(dev, x, *tables, B, T, C, HW)
            assert same_bits(got, E.tsf_tokens_ref(x, *tables)), f"{dtype} x, tables {[t is not None for t in tables]}"
        back = Guarded(dev, (B, T, C, HW), dtype)
        _ops().tsf_untokenize(got, back.t, B, T, C, HW)
        want = got.reshape(B, HW, T, C).permute(0, 2, 3, 1).to(dtype)
        assert same_bits(back.written(f"untokenize to {dtype}"), want), f"untokenize to {dtype}"


@pytest.mark.parametrize("C,HW", [(33, 31), (768, 49)])
def test_untokenize_to_f16_overflows_and_rounds_like_torch(dev, C, HW):
    """bf16 tokens beyond f16's range become +-inf (65280 is the last finite bf16 below f16's 65504, 65536 overflows),
    tiny ones f16 subnormals or zero: the same bits as torch's bf16 -> f16 cast."""
    B, T = 2, 3
    g = torch.Generator(device=dev).manual_seed(C + HW)
    tok = torch.randn(B * HW * T, C, generator=g, device=dev)
    special = torch.tensor([65280.0, 65536.0, -65536.0, 1e5, -3e38, 6e-8, 3e-8, -1e-6, 1e-10, -0.0, 65504.0, 2.0 ** -24],
                           device=dev)
    pick = torch.randint(0, special.numel(), tok.shape, generator=g, device=dev)
    tok = torch.where(torch.rand(tok.shape, generator=g, device=dev) < 0.3, special[pick], tok).to(bf16)
    back = Guarded(dev, (B, T, C, HW), f16)
    _ops().tsf_untokenize(tok, back.t, B, T, C, HW)
    want = tok.reshape(B, HW, T, C).permute(0, 2, 3, 1).to(f16)
    assert bool(torch.isinf(want).any()) and bool((want != 0).logical_and(want.abs() < 2.0 ** -14).any())
    back.guards("untokenize to f16")
    assert same_bits(back.t, want)
