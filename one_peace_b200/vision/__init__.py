"""The vision branch's backbones: the ImageNet classifier (one_peace_vision/classification: ``models_vit`` and the criteria
of ``main_ft.py``), the detection backbone (``det``), the action-recognition backbone (``video``), the segmentation
backbone (``seg``) and its multi-scale deformable attention (``ms_deform_attn.MSDeformAttn``)."""
import torch
import torch.nn.functional as F


def _get_rank():
    if torch.distributed.is_available() and torch.distributed.is_initialized():
        return torch.distributed.get_rank()
    return 0


def resize_abs_pos_embed(self, checkpoint):
    """The ``resize_abs_pos_embed`` method of the detection and recognition backbones (det/models/onepeace.py:535-558,
    video/mmaction_custom/models/backbones/onepeace.py:526-551): bicubic resize of the checkpoint's positional rows onto
    ``self.image_adapter``'s bucket grid, the first row kept."""
    pos = checkpoint["image_adapter.pos_embed"]
    dim = pos.shape[-1]
    num_patches = self.image_adapter.bucket_size ** 2
    extra = self.image_adapter.pos_embed.shape[-2] - num_patches
    orig, new = int((pos.shape[-2] - extra) ** 0.5), int(num_patches ** 0.5)
    if orig != new:
        if _get_rank() == 0:
            print(f"Position interpolate from {orig}x{orig} to {new}x{new}")
        tok = pos[extra:].reshape(-1, orig, orig, dim).permute(0, 3, 1, 2)
        tok = F.interpolate(tok, size=(new, new), mode="bicubic", align_corners=False)
        checkpoint["image_adapter.pos_embed"] = torch.cat((pos[:extra], tok.permute(0, 2, 3, 1).flatten(0, 2)), dim=0)
