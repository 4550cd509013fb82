"""CPU: the fp64 references of the segmentation kernels (tests/seg_ref.py) equal torch's own depthwise conv + GELU,
bilinear resize and transposed conv, on square, non-square and odd grids."""
import pytest
import torch
import torch.nn.functional as F

import seg_ref as R

SHAPES = [[(8, 8), (4, 4), (2, 2)], [(6, 10), (3, 5), (2, 3)], [(7, 5)], [(1, 1), (3, 1)]]


@pytest.mark.parametrize("shapes", SHAPES)
@pytest.mark.parametrize("B", [1, 2])
def test_dwconv_gelu_matches_torch(shapes, B):
    g = torch.Generator().manual_seed(0)
    C = 16
    T = sum(h * w for h, w in shapes)
    x = torch.randn(B * T, C, generator=g, dtype=torch.float64)
    w = torch.randn(C, 1, 3, 3, generator=g, dtype=torch.float64)
    b = torch.randn(C, generator=g, dtype=torch.float64)
    y, _, _ = R.dwconv_gelu_ref(x, w, b, shapes, B)
    want = R._rows([F.gelu(F.conv2d(lv, w, b, padding=1, groups=C)) for lv in R._levels(x, shapes, B)])
    torch.testing.assert_close(y, want, rtol=0, atol=1e-12)


@pytest.mark.parametrize("hw,g", [((16, 16), 4), ((8, 8), 4), ((4, 4), 4), ((2, 2), 4), ((12, 20), 5), ((7, 3), 5)])
def test_bilinear_matches_interpolate(hw, g):
    x = torch.randn(2, 3, g, g, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    got, _ = R.bilinear_ref(x, *hw)
    torch.testing.assert_close(got, F.interpolate(x, size=hw, mode="bilinear", align_corners=False), rtol=0, atol=1e-12)


def test_bilinear_scale_factors_match_the_reference_calls():
    """onepeace_adapter.py:125-127 resizes by scale_factor 4, 2 and 0.5; x 1/2 is a 2 x 2 mean."""
    x = torch.randn(1, 2, 6, 6, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    for f in (4, 2, 0.5):
        n = int(6 * f)
        torch.testing.assert_close(R.bilinear_ref(x, n, n)[0],
                                   F.interpolate(x, scale_factor=f, mode="bilinear", align_corners=False), rtol=0, atol=1e-12)
    torch.testing.assert_close(R.bilinear_ref(x, 3, 3)[0], F.avg_pool2d(x, 2), rtol=0, atol=1e-12)


@pytest.mark.parametrize("hw", [(4, 4), (3, 5)])
def test_convt_matches_conv_transpose2d(hw):
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 6, *hw, generator=g, dtype=torch.float64)
    w = torch.randn(6, 5, 2, 2, generator=g, dtype=torch.float64)
    b = torch.randn(5, generator=g, dtype=torch.float64)
    torch.testing.assert_close(R.convt_ref(x, w, b), F.conv_transpose2d(x, w, b, stride=2), rtol=0, atol=1e-12)
