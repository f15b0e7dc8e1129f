"""The sliced parity rule (tests/slice_parity.py) on synthetic outputs: independent noise at the oracle's own level
passes, a 3 % error in one slice fails where the whole-output gate passes, the floor keeps slices with no 16-bit error of
their own from failing on noise, and the index-sampled form of the large golden cases finds the same (sample, frame)."""
import pytest
import torch

from tests.slice_parity import assert_sliced_parity, sliced_parity

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
