"""Float64 restatement of the ImageNet loader's transforms (turboprune_b200.utils.dataset, tp_resized_crop).

* ``resized_crop``: the box alone, ``F.interpolate(antialias=True)`` in float64 (PIL's bilinear filter), the flip,
  then ``(v - mean255) / std255`` with the reference's float64 constants (utils/dataset.py:28-29).
* ``rrc_box``: torchvision's ``RandomResizedCrop.get_params`` for one image, statement by statement, with the random
  draws replaced by given uniforms (area, log-aspect and offset draws in [0, 1)).
* ``center_box``: FFCV's ``get_center_crop`` (CenterCropRGBImageDecoder).
"""
import math

import torch
import torch.nn.functional as F

MEAN255 = torch.tensor([0.485, 0.456, 0.406], dtype=torch.float64) * 255
STD255 = torch.tensor([0.229, 0.224, 0.225], dtype=torch.float64) * 255


def resized_crop(img, box, flip, size=224):
    """img uint8 [3, H, W] (any device) -> float64 [3, size, size] on the CPU."""
    t, l, h, w = (int(v) for v in box)
    crop = img[:, t:t + h, l:l + w].cpu().double()[None]
    r = F.interpolate(crop, (size, size), mode="bilinear", antialias=True, align_corners=False)[0]
    if flip:
        r = r.flip(-1)
    return (r - MEAN255.view(3, 1, 1)) / STD255.view(3, 1, 1)


def rrc_box(height, width, u_area, u_ratio, u_off, scale=(0.08, 1.0), ratio=(3 / 4, 4 / 3)):
    area = height * width
    log_ratio = (math.log(ratio[0]), math.log(ratio[1]))
    for k in range(10):
        target_area = area * (scale[0] + (scale[1] - scale[0]) * float(u_area[k]))
        aspect_ratio = math.exp(log_ratio[0] + (log_ratio[1] - log_ratio[0]) * float(u_ratio[k]))
        w = int(round(math.sqrt(target_area * aspect_ratio)))
        h = int(round(math.sqrt(target_area / aspect_ratio)))
        if 0 < w <= width and 0 < h <= height:
            i = int(math.floor(float(u_off[0]) * (height - h + 1)))
            j = int(math.floor(float(u_off[1]) * (width - w + 1)))
            return i, j, h, w
    in_ratio = float(width) / float(height)
    if in_ratio < min(ratio):
        w = width
        h = int(round(w / min(ratio)))
    elif in_ratio > max(ratio):
        h = height
        w = int(round(h * max(ratio)))
    else:
        w = width
        h = height
    return (height - h) // 2, (width - w) // 2, h, w


def center_box(height, width, ratio=224 / 256):
    c = int(ratio * min(height, width))
    return (height - c) // 2, (width - c) // 2, c, c
