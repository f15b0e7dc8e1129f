"""Open-Sora-Plan v1.2.0 with a conv down-sampler (``downsampler="k333_s222"`` / ``"k33_s22"``): the front end's host logic on
the torch stand-ins of the kernels (tests/kernels_emul.py, tests/kernels_emul_ds.py), fp32, against the outputs of the UNMODIFIED reference model stored
in tests/golden/osp_v120_ds.pt (oracle/gen_golden_osp_ds.py), the state-dict layout against the reference, and the
configurations the reference cannot run."""
import os

import pytest
import torch

from oracle import osp_cases as OC, ref_loader
from oracle.gen_golden_osp_ds import CASES12_DS, inputs_ds, weights_ds
from tests import kernels_emul_ds
from videosys_b200.models.transformers.open_sora_plan_v120_transformer_3d import OpenSoraT2V


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "osp_v120_ds.pt"))


def _net(name):
    net = OpenSoraT2V(**CASES12_DS[name][0])
    net.load_state_dict(weights_ds(net.state_dict(), name, torch.float32))
    return net.eval()


def _call(net, x, enc, m, t, **kw):
    return net(x, timestep=t, encoder_hidden_states=enc, encoder_attention_mask=m, return_dict=False, **kw)[0]


@pytest.mark.parametrize("name", ["ds3_rope", "ds3_abspos", "ds2_rope"])
def test_osp_v120_downsampler_host_logic_vs_reference_golden(monkeypatch, gold, name):
    kernels_emul_ds.emulate(monkeypatch)
    out = _call(_net(name), *inputs_ds(name, torch.float32))
    want = gold[f"{name}.fp32"]
    assert out.shape == want.shape
    assert torch.allclose(out, want, rtol=1e-4, atol=1e-5), (out - want).abs().max()


def test_osp_v120_downsampler_pab_steps_vs_reference_golden(monkeypatch, gold):
    """Eight PAB steps (spatial + cross broadcast): the cached attention output stays in the sub-grid order and is replayed
    through the un-shuffling gate + residual."""
    from videosys_b200.core.pab import pab_mgr

    kernels_emul_ds.emulate(monkeypatch)
    net = _net("ds3_rope")
    pab_mgr.set_pab_manager(pab_mgr.PABConfig(**OC.PAB12_KW))
    pab_mgr.update_steps(len(OC.PAB_TIMESTEPS))
    net.reset_pab_state()
    try:
        for step, t in enumerate(OC.PAB_TIMESTEPS):
            x, enc, m, _ = inputs_ds("ds3_rope", torch.float32, step)
            out = _call(net, x, enc, m, torch.tensor([t, t]), ts_int=t)
            want = gold[f"pab.{step}.fp32"]
            assert torch.allclose(out, want, rtol=1e-4, atol=1e-5), (step, (out - want).abs().max())
    finally:
        pab_mgr.set_pab_manager(None)


@pytest.mark.parametrize("name", ["ds3_rope", "ds2_rope"])
def test_osp_v120_downsampler_state_dict_matches_reference(name):
    if not ref_loader.available():
        pytest.skip("reference checkout not present")
    cfg = CASES12_DS[name][0]
    ref = ref_loader.build_osp_v120(dtype=torch.float32, **cfg)
    ours = OpenSoraT2V(**cfg)
    rs, os_ = ref.state_dict(), ours.state_dict()
    assert {k: tuple(v.shape) for k, v in rs.items()} == {k: tuple(v.shape) for k, v in os_.items()}
    ours.load_state_dict(weights_ds(rs, name, torch.float32), strict=True)
    ref.load_state_dict(ours.state_dict(), strict=True)


def test_osp_v120_downsampler_state_dict_names():
    """The reference's parameter names and shapes (:653-682, :1033-1088, :372-400) for one block and the patch embedding."""
    C = 192
    sd = OpenSoraT2V(**CASES12_DS["ds3_rope"][0]).state_dict()
    want = {"pos_embed.proj.weight": (C, 4, 1, 2, 2), "transformer_blocks.0.attn1.downsampler.layer.weight": (C, 1, 3, 3, 3),
            "transformer_blocks.0.attn1.downsampler.layer.bias": (C,), "transformer_blocks.0.ff.project_in.weight": (2 * C, C),
            "transformer_blocks.0.ff.dwconv.0.weight": (2 * C, 1, 5, 5), "transformer_blocks.0.ff.dwconv.1.weight": (2 * C, 1, 3, 3),
            "transformer_blocks.0.ff.dwconv.2.weight": (2 * C, 1, 1, 1), "transformer_blocks.0.ff.dwconv.2.bias": (2 * C,),
            "transformer_blocks.0.ff.project_out.weight": (C, 2 * C)}
    assert {k: tuple(sd[k].shape) for k in want} == want
    assert not any(".ff.net." in k for k in sd)
    sd2 = OpenSoraT2V(**CASES12_DS["ds2_rope"][0]).state_dict()
    assert tuple(sd2["pos_embed.proj.weight"].shape) == (C, 4, 2, 2)
    assert tuple(sd2["transformer_blocks.0.attn1.downsampler.layer.weight"].shape) == (C, 1, 3, 3)


def test_osp_v120_downsampler_rejections(monkeypatch):
    kernels_emul_ds.emulate(monkeypatch)
    with pytest.raises(ValueError, match="does not divide"):  # 6 x 10 latent pixels = 3 x 5 patches, down factor 2
        cfg, _, L, _ = CASES12_DS["ds3_rope"]
        net = _net("ds3_rope")
        _call(net, torch.zeros(2, 4, 4, 6, 10), torch.zeros(2, 1, L, 32), torch.ones(2, 1, L), torch.tensor([500, 500]))
    with pytest.raises(ValueError, match="one latent frame"):
        _call(_net("ds2_rope"), torch.zeros(2, 4, 4, 8, 8), torch.zeros(2, 1, 7, 32), torch.ones(2, 1, 7), torch.tensor([500, 500]))
    base = CASES12_DS["ds3_rope"][0]
    for spec in ("k533_s222", "k373_s222", "k77_s22"):
        with pytest.raises(NotImplementedError):
            OpenSoraT2V(**dict(base, downsampler=spec))
    with pytest.raises(NotImplementedError, match="sequence parallelism"):
        _net("ds3_rope").enable_parallel(dp_size=1, sp_size=2)
