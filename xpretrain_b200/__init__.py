"""xpretrain_b200 — H100-native (sm_90a) implementation of the XPretrain video-text dual-encoder hot path.

Public surface mirrors the reference's CLIP-ViP entry points (SURVEY.md §8b):
  xpretrain_b200.modeling.VidCLIP            <- CLIP-ViP/src/modeling/VidCLIP.py
  xpretrain_b200.optimization.loss           <- CLIP-ViP/src/optimization/loss.py (NCELearnableTempLoss, build_loss_func)
  xpretrain_b200.utils.distributed.allgather <- hvd.allgather (run_pretrain.py:344-345)
Everything computes in hand-written CUDA behind the C ABI in include/xpretrain_b200.h; importing the package
does not need a GPU, calling it does.
"""
__version__ = "0.1.0"
