"""The temporal VAE's decode planner (temporal_vae.decode_plan / decode_peak_bytes): pure shape arithmetic, no device."""
import pytest

from star_b200.video_to_video.modules.temporal_vae import PASS_BYTES, DecodePlan, _pass_bytes, _stages, decode_peak_bytes, \
    decode_plan

GiB = 1 << 30
FULL = (128, 256, 512, 512)

# (bf, num_frames, latent h, latent w, block_out_channels): the bench's VAE sweep (540p/720p, 960p, 1080p outputs), the denoise
# bench's decode, and the shapes the test suite decodes
TRIVIAL = [(3, 3, 90, 160, FULL), (3, 3, 122, 216, FULL), (3, 3, 138, 248, FULL), (2, 2, 122, 216, FULL),
           (3, 3, 14, 16, FULL), (3, 3, 10, 12, (64, 64, 128, 128)), (6, 3, 4, 6, (64, 64, 128, 128)),
           (2, 2, 4, 6, (64, 64, 128, 128)), (3, 3, 330, 330, (32, 32, 64, 64))]


@pytest.mark.parametrize("bf,T,h,w,ch", TRIVIAL)
def test_bench_and_test_shapes_get_the_trivial_plan(bf, T, h, w, ch):
    assert decode_plan(bf, T, h, w, ch) == DecodePlan(bf, h * w * 64, h * 8)


@pytest.mark.parametrize("h,w", [(362, 648), (546, 968)], ids=["720p_to_4x", "1080p_to_4x"])
def test_4x_windows_get_split_plans_within_the_budget(h, w):
    plan = decode_plan(3, 3, h, w)
    assert plan.frames < 3 and plan.band < h * w * 64 and plan.rows < h * 8 and plan.rows % 2 == 0
    assert max(max(_pass_bytes(plan.frames, plan.rows, *s)) for s in _stages(h, w, FULL, 2)) <= PASS_BYTES
    assert decode_peak_bytes(plan, 3, h, w) < decode_peak_bytes(DecodePlan(3, h * w * 64, h * 8), 3, h, w)


def test_1080p_to_4x_window_predicted_with_margin_under_the_card():
    """the window's activations plus the pipeline's resident weights (4.2 GiB: UNet + VAE) stay 7 GiB under the 79.2 GiB an
    80 GB H100 gives to PyTorch, room for the caching allocator's fragmentation"""
    plan = decode_plan(3, 3, 546, 968)
    assert plan.frames == 1
    assert decode_peak_bytes(plan, 3, 546, 968) + 4.2 * GiB <= 72.2 * GiB


def test_plans_are_deterministic_and_shape_only():
    shapes = [(3, 3, 546, 968), (3, 3, 362, 648), (2, 2, 546, 968), (1, 1, 546, 968), (3, 3, 90, 160)]
    assert [decode_plan(*s) for s in shapes] == [decode_plan(*s) for s in reversed(shapes)][::-1]
    for s in shapes:
        p = decode_plan(*s)
        assert p.frames >= 1 and p.band >= 128 and p.rows >= 2 and decode_plan(*s) == p


def test_plan_rejects_a_ragged_window():
    with pytest.raises(ValueError):
        decode_plan(4, 3, 16, 24)
