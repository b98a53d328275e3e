"""Tile geometry of spatially tiled sampling (video_to_video_model.make_tiles): coverage, equal tile shapes, real overlap,
and blend weights that form a partition of unity."""
import pytest
import torch

from star_b200.video_to_video.video_to_video_model import make_tiles


def coverage(ranges, length):
    n = torch.zeros(length, dtype=torch.int64)
    for s, e in ranges:
        n[s:e] += 1
    return n


def weight_sum(ranges, weights, length):
    total = torch.zeros(length, dtype=torch.float64)
    for (s, e), w in zip(ranges, weights):
        total[s:e] += w.double()
    return total


CASES = [
    # h, w, tile, overlap
    (362, 648, (90, 160), 16),
    (242, 432, (90, 160), 16),
    (122, 216, (90, 160), 16),
    (42, 48, (26, 32), 8),
    (91, 161, (90, 160), 16),          # L = T + 1 on both axes
    (50, 100, (90, 160), 16),          # both axes shorter than the tile
    (90, 160, (90, 160), 16),          # exactly one tile
    (122, 216, (34, 40), 0),           # no ramp: overlaps left by the even spread are shared equally
    (362, 648, (58, 64), 40),          # wide ramps
]


@pytest.mark.parametrize("h,w,tile,overlap", CASES)
def test_tiles_cover_every_pixel_with_equal_shapes(h, w, tile, overlap):
    rows, cols, row_w, col_w = make_tiles(h, w, tile, overlap)
    for ranges, length, t, weights in ((rows, h, tile[0], row_w), (cols, w, tile[1], col_w)):
        assert ranges[0][0] == 0 and ranges[-1][1] == length
        assert (coverage(ranges, length) >= 1).all()
        size = min(length, t)
        assert all(e - s == size for s, e in ranges)
        assert all(0 <= s < e <= length for s, e in ranges)
        assert [s for s, _ in ranges] == sorted({s for s, _ in ranges})
        for (s0, e0), (s1, _) in zip(ranges, ranges[1:]):
            assert e0 - s1 >= overlap, f"real overlap {e0 - s1} < requested {overlap}"
        if length > t:
            assert len(ranges) == -(-(length - t) // (t - overlap)) + 1
        else:
            assert len(ranges) == 1
        assert len(weights) == len(ranges)
        assert all(wt.dtype == torch.float32 and wt.shape == (size,) for wt in weights)


@pytest.mark.parametrize("h,w,tile,overlap", CASES)
def test_weights_are_a_partition_of_unity(h, w, tile, overlap):
    rows, cols, row_w, col_w = make_tiles(h, w, tile, overlap)
    for ranges, weights, length in ((rows, row_w, h), (cols, col_w, w)):
        assert all((wt > 0).all() for wt in weights)
        assert torch.allclose(weight_sum(ranges, weights, length), torch.ones(length, dtype=torch.float64), rtol=0, atol=1e-6)
        once = coverage(ranges, length) == 1
        for (s, e), wt in zip(ranges, weights):
            single = once[s:e]
            assert (wt[single] == 1.0).all(), "a pixel covered by one tile must have weight exactly 1.0"
    # 2-D: products of the per-axis weights also sum to 1 at every pixel
    total = torch.zeros(h, w, dtype=torch.float64)
    for (r0, r1), wy in zip(rows, row_w):
        for (c0, c1), wx in zip(cols, col_w):
            total[r0:r1, c0:c1] += wy.double()[:, None] * wx.double()[None, :]
    assert torch.allclose(total, torch.ones_like(total), rtol=0, atol=2e-6)


def test_single_tile_has_unit_weights():
    rows, cols, row_w, col_w = make_tiles(42, 48, (50, 64), 16)
    assert rows == [(0, 42)] and cols == [(0, 48)]
    assert torch.equal(row_w[0], torch.ones(42)) and torch.equal(col_w[0], torch.ones(48))


def test_ramp_shape_at_inner_edges():
    """two tiles of 26 over 42 rows, overlap 8: starts 0 and 16 (real overlap 10); the ramps rise over 8 pixels from the
    inner edges, and the outer edges keep weight 1"""
    rows, _, row_w, _ = make_tiles(42, 48, (26, 48), 8)
    assert rows == [(0, 26), (16, 42)]
    first, second = row_w[0].double(), row_w[1].double()
    assert (first[:16] == 1.0).all() and (second[10:] == 1.0).all()
    assert (first[16:].diff() < 0).all() and (second[:10].diff() > 0).all()


@pytest.mark.parametrize("tile,overlap", [
    ((88, 160), 16),     # th != 2 (mod 8)
    ((90, 164), 16),     # tw != 0 (mod 8)
    ((0, 160), 16),
    ((-6, 160), 0),
    ((90, 0), 0),
    ((90, 160), -1),
    ((90, 160), 90),     # overlap >= th
    ((26, 16), 16),      # overlap >= tw
])
def test_bad_tiles_raise(tile, overlap):
    with pytest.raises(ValueError):
        make_tiles(362, 648, tile, overlap)
