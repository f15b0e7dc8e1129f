"""The sliced parity rule (tests/slice_parity.py) on synthetic outputs: independent noise at the oracle's own level
passes, a 3 % error in one slice fails where the whole-output gate passes, the floor keeps slices with no 16-bit error of
their own from failing on noise, and the index-sampled form of the large golden cases finds the same (sample, frame).
The same for the 2-D pixel tiles of image-shaped outputs, where an error along one vertical seam fails the tiles that
the row bands and the whole-output gate pass, and partial edge tiles hold each element once."""
import pytest
import torch

from tests.slice_parity import _tile_sq_hw, assert_sliced_parity, sliced_parity

B, T, H, W, C = 2, 6, 15, 20, 256  # 300 tokens per frame: two full 128-row tiles and a ragged one
REL = 1e-2  # the 16-bit oracle's own relative error at the real widths


def _outputs(seed=0):
    """(ours, r16, r32) as [B, T, N, C]: r16 and ours each r32 plus independent noise of relative size REL."""
    g = torch.Generator().manual_seed(seed)
    r32 = torch.randn(B, T, H * W, C, generator=g, dtype=torch.float64)
    r16 = r32 + REL * r32.abs() * torch.randn(r32.shape, generator=g, dtype=torch.float64)
    ours = r32 + REL * r32.abs() * torch.randn(r32.shape, generator=g, dtype=torch.float64)
    return ours, r16, r32


def _latent(x):
    """[B, T, N, C] -> the [B, C, T, H, W] layout of a latent (axes "bctnn")."""
    return x.view(B, T, H, W, C).permute(0, 4, 1, 2, 3).contiguous()


def test_noise_at_the_oracle_level_passes():
    ours, r16, r32 = _outputs()
    rep = assert_sliced_parity("synthetic noise", ours, r16, r32, "btnc")
    assert rep.grid == (B, T, 3, 2) and rep.tile == (128, 128)
    assert rep.worst < 0.9 and rep.old_gate_ok


def test_narrow_output_slices_keep_the_channels_together():
    """An 8-channel output: slices of 2048 tokens x all 8 channels, as many elements as a 128 x 128 tile."""
    ours, r16, r32 = (v.reshape(B, T, H * W * C // 8, 8) for v in _outputs(5))
    rep = assert_sliced_parity("synthetic narrow", ours, r16, r32, "btnc")
    assert rep.tile == (2048, 8) and rep.grid == (B, T, 5, 1)


def test_floor_covers_slices_without_an_own_error():
    """A frame where the 16-bit oracle is exact (r16 == r32) and ours carries rounding noise far below the output's own
    error: only the floor lets it pass, and it does."""
    ours, r16, r32 = _outputs(1)
    r16[0, 2] = r32[0, 2]
    ours[0, 2] = r32[0, 2] + 1e-3 * REL * r32[0, 2].abs() * torch.randn(r32[0, 2].shape, dtype=torch.float64)
    assert_sliced_parity("synthetic exact frame", ours, r16, r32, "btnc")
    ours[0, 2] = r32[0, 2] + REL * r32[0, 2].abs()  # a real error there still fails
    assert not sliced_parity("synthetic exact frame, real error", ours, r16, r32, "btnc").ok


@pytest.mark.parametrize("layout", ["btnc", "bctnn"])
def test_three_percent_in_one_slice_fails_where_the_whole_output_gate_passes(layout):
    ours, r16, r32 = _outputs(2)
    ours[1, 3, 128:256, 128:256] += 0.03 * r32[1, 3, 128:256, 128:256]
    if layout == "bctnn":
        ours, r16, r32 = _latent(ours), _latent(r16), _latent(r32)
    rep = sliced_parity("synthetic 3 % slice", ours, r16, r32, layout)
    print(rep.describe())
    assert rep.old_gate_ok, "the whole-output gate should not see a 3 % error in 1/72 of the output"
    assert not rep.ok and rep.worst > 2.0
    assert rep.worst_at == (1, 3, 128, 128)


@pytest.mark.parametrize("layout", ["btnc", "bctnn"])
def test_index_sampled_form_finds_the_same_frame(layout):
    ours, r16, r32 = _outputs(3)
    bad = ours.clone()
    bad[1, 3, 128:256, 128:256] += 0.03 * r32[1, 3, 128:256, 128:256]
    if layout == "bctnn":
        ours, bad, r16, r32 = _latent(ours), _latent(bad), _latent(r16), _latent(r32)
    shape = tuple(r32.shape)
    idx = torch.randperm(r32.numel(), generator=torch.Generator().manual_seed(4))[: r32.numel() // 5]
    pick = lambda x: x.flatten()[idx]  # noqa: E731
    good = assert_sliced_parity("synthetic noise, sampled", pick(ours), pick(r16), pick(r32), layout, idx=idx, shape=shape)
    assert good.grid == (B, T, 1, 1)
    rep = sliced_parity("synthetic 3 % slice, sampled", pick(bad), pick(r16), pick(r32), layout, idx=idx, shape=shape)
    print(rep.describe())
    assert not rep.ok and rep.worst_at[:2] == (1, 3)
    assert rep.old_gate_ok


# ---- image-shaped outputs: 2-D pixel tiles (axes h / w) -----------------------------------------------------------------
def _video(shape, seed):
    """(ours, r16, r32) as [B, 3, T, H, W] float32: r16 and ours each r32 plus independent noise of relative size REL."""
    g = torch.Generator().manual_seed(seed)
    r32 = torch.randn(shape, generator=g)
    r16 = r32 + REL * r32.abs() * torch.randn(shape, generator=g)
    ours = r32 + REL * r32.abs() * torch.randn(shape, generator=g)
    return ours, r16, r32


def test_pixel_tiles_noise_at_the_oracle_level_passes():
    ours, r16, r32 = _video((2, 3, 5, 150, 200), 6)
    rep = assert_sliced_parity("synthetic video noise", ours, r16, r32, "bcthw")
    assert rep.grid == (2, 5, 3, 4, 1) and rep.tile == (64, 64, 3)
    assert rep.worst < 0.9 and rep.old_gate_ok


def test_one_blend_zone_strip_fails_pixel_tiles_where_row_bands_and_the_whole_output_pass():
    """A 3 % error in one 64-column strip (the width of a tiled decode's blend zone) of one frame of a 49 x 480 x 720 RGB
    video: a fraction 64 / 720 of every row band, and 1 / 551 of the output, but the whole of a column of 2-D tiles."""
    ours, r16, r32 = _video((1, 3, 49, 480, 720), 7)
    ours[0, :, 20, :, 320:384] += 0.03 * r32[0, :, 20, :, 320:384]
    whole_and_bands = sliced_parity("synthetic strip, row bands", ours, r16, r32, "bctnn")
    print(whole_and_bands.describe())
    assert whole_and_bands.old_gate_ok and whole_and_bands.ok
    rep = sliced_parity("synthetic strip, pixel tiles", ours, r16, r32, "bcthw")
    print(rep.describe())
    assert not rep.ok and rep.worst > 1.5
    assert rep.worst_at[:2] == (0, 20) and rep.worst_at[3] == 320
    assert bool((rep.loads[0, 20, :, 5] > 1.5).all()) and rep.loads[0, 20].max(dim=0).values.sort().values[-2] < 1.0


def test_pixel_tiles_floor_covers_a_flat_tile():
    """A near-zero 64 x 64 tile where the 16-bit oracle is exact and ours carries noise far below the output's own error:
    the floor lets it pass; a real error there fails."""
    ours, r16, r32 = _video((1, 3, 4, 128, 192), 8)
    r32[0, :, 1, 64:128, 64:128] *= 1e-3
    r16[0, :, 1, 64:128, 64:128] = r32[0, :, 1, 64:128, 64:128]
    flat = r32[0, :, 1, 64:128, 64:128]
    ours[0, :, 1, 64:128, 64:128] = flat + 1e-3 * REL * flat.abs() * torch.randn(flat.shape)
    rep = assert_sliced_parity("synthetic flat tile", ours, r16, r32, "bcthw")
    assert float(rep.ratios[0, 1, 1, 1, 0]) > 1e3  # far above its own error: only the floor passes it
    ours[0, :, 1, 64:128, 64:128] = flat + 0.3 * r32[0, :, 1].abs().mean()
    assert not sliced_parity("synthetic flat tile, real error", ours, r16, r32, "bcthw").ok


def test_partial_edge_tiles_are_counted_once():
    """100 x 150 pixels: tiles of 64 and 36 rows by 64, 64 and 22 columns.  Every element lands in exactly one tile, and
    an error in the bottom-right corner is found in the partial tile that holds it."""
    counts = _tile_sq_hw(torch.ones(1, 2, 100, 150, 3, dtype=torch.float64), 64, 64, 3)
    assert counts.shape == (1, 2, 2, 3, 1)
    rows, cols = torch.tensor([64.0, 36.0]), torch.tensor([64.0, 64.0, 22.0])
    assert torch.equal(counts[0, 0, :, :, 0], 3 * rows[:, None] * cols[None, :].double())
    assert float(counts.sum()) == 2 * 100 * 150 * 3
    ours, r16, r32 = _video((1, 3, 2, 100, 150), 9)
    ours[0, :, 1, 90:, 140:] += 0.2 * r32[0, :, 1, 90:, 140:]
    rep = sliced_parity("synthetic edge tiles, corner error", ours, r16, r32, "bcthw")
    print(rep.describe())
    assert rep.grid == (1, 2, 2, 3, 1)
    assert not rep.ok and rep.worst_at == (0, 1, 64, 128, 0)
