"""CPU: the gradient-checkpointing switches of CLIPModel carry the reference's names (CLIP_ViP.py:478,524-526,626) and change
neither the parameters nor the absence of a CPU path."""
import pytest
import torch

from clipvip_cases import b16, vidclip


def _vidclip():
    return vidclip(b16(1, 1))


def test_switches_have_the_reference_names_and_default_off():
    from xpretrain_b200.modeling.clip_vip import CLIPModel
    assert CLIPModel.supports_gradient_checkpointing is True
    cm = _vidclip().clipmodel
    encoders = (cm.vision_model.encoder, cm.text_model.encoder)
    assert all(enc.gradient_checkpointing is False for enc in encoders)
    assert cm.is_gradient_checkpointing is False
    cm.gradient_checkpointing_enable()
    assert all(enc.gradient_checkpointing is True for enc in encoders)
    assert cm.is_gradient_checkpointing is True
    cm.gradient_checkpointing_disable()
    assert all(enc.gradient_checkpointing is False for enc in encoders)
    assert cm.is_gradient_checkpointing is False
    cm.gradient_checkpointing_enable(gradient_checkpointing_kwargs={"use_reentrant": False})   # Hugging Face call sites
    assert cm.is_gradient_checkpointing is True
    cm.vision_model.encoder.gradient_checkpointing = False          # the reference attribute, set on one encoder
    assert cm.is_gradient_checkpointing is True
    with pytest.raises(AttributeError):
        cm.is_gradient_checkpointing = False


def test_switches_leave_the_state_dict_unchanged():
    model = _vidclip()
    before = {k: (tuple(v.shape), v.dtype) for k, v in model.state_dict().items()}
    model.clipmodel.gradient_checkpointing_enable()
    after = {k: (tuple(v.shape), v.dtype) for k, v in model.state_dict().items()}
    assert after == before


def test_checkpointed_cpu_forward_still_raises():
    from xpretrain_b200 import _lib
    model = _vidclip()
    model.clipmodel.gradient_checkpointing_enable()
    model.train()
    with pytest.raises(_lib.XpError):
        model(video=torch.zeros(1, 1, 3, 224, 224), text_input_ids=torch.zeros(1, 4, dtype=torch.long),
              text_input_mask=torch.ones(1, 4, dtype=torch.long))
