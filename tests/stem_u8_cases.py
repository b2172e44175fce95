"""Shape tables and normalisations of the uint8 stem tests (test_stem_u8_gpu.py), on top of
tail_cases.py.  The uint8 kernels stage a tile with 4-byte cp.async when W % 4 == 0 (a row is 3W
bytes) and element by element otherwise; the CPU suite checks that these tables reach both paths,
odd 3W, cut tiles and the multi-tile walk."""
import torch

import tail_cases as tc

StemCase = tc.StemCase

# torchvision's ImageNet statistics, and inception's 0.5 / 0.5 (reference utils/dataflow.py)
NORMS = {
    "imagenet": ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225)),
    "inception": ((0.5, 0.5, 0.5), (0.5, 0.5, 0.5)),
}


def host_normalize(u, norm):
    """bf16(Normalize(mean, std)(ToTensor()(u))) on the CPU, in u's HWC layout: the fp32
    operations of torchvision's transforms, then the bf16 cast."""
    mean = torch.tensor(norm[0], dtype=torch.float32)
    std = torch.tensor(norm[1], dtype=torch.float32)
    return u.cpu().float().div(255).sub(mean).div(std).to(torch.bfloat16)


def u8_aligned(W):
    """The uint8 staging path: 4-byte words when the 3W-byte rows are 4-byte aligned."""
    return W % 4 == 0


# W % 4 == 0 widths: 44 (one tile column), 68 (two, cut), 224 (the training size), 4 and 8 (one or
# two output pixels per row)
U8_CASES = [StemCase(2, 38, 44, co) for co in tc.STEM_FWD_COUT] + [
    StemCase(3, 36, 68, 32), StemCase(2, 224, 224, 32), StemCase(2, 3, 4, 16), StemCase(1, 4, 4, 8),
    StemCase(2, 5, 8, 64),
]
# 228 x 228 -> 114 x 114 outputs: 66 x 8 x 4 = 2112 tiles = 2 x 8 x 132, last tile row and column cut
U8_WALK_CASES = [StemCase(66, 228, 228, co) for co in tc.STEM_WGRAD_COUT]

DIRECT_CASES = tc.STEM_CASES + U8_CASES
WALK_CASES = tc.STEM_WALK_CASES + U8_WALK_CASES
EVAL_SHAPES = tc.STEM_EVAL_SHAPES + ((2, 38, 44),)
