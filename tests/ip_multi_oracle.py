"""Image-prompt sets (DESIGN.md §13) for the f32 CPU oracle, whose attn2 takes several prompts, each unmasked (one softmax over
all its tokens) or masked (one softmax per image, weighted per query by the image's mask downsampled as diffusers'
IPAdapterMaskProcessor.downsample does; oracle/unet_oracle.py). Here: the masks' binarisation."""
from __future__ import annotations

from typing import Optional

import torch


def binarize(mask: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    """diffusers' mask processor binarisation at 0.5 (what set_image_prompts applies)."""
    return None if mask is None else (mask.float() >= 0.5).float()
