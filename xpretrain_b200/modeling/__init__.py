from .clip_vip import CLIPModel, ClipVipConfig, TowerConfig  # noqa: F401
from .vidclip import VidCLIP  # noqa: F401
from .lfvila import LFVILA_Video_Classification  # noqa: F401
