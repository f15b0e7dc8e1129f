"""STDiT3 in FP8 mode (set_fp8_linears) on the H100 at the full OpenSora width (hidden 1152, 16 heads): the velocity
against the bf16 forward (a wrong scale, a swapped weight or a missed row shows as a relative L2 distance of order 1; the
quantization of the six block Linears stays below 0.1), the mode toggled off reproducing the bf16 output bit for bit,
and a PAB sampling run whose replayed step graphs equal the eager steps bit for bit."""
import pytest
import torch

from oracle import cases, synth
from videosys_b200.core.graph_step import StepGraph
from videosys_b200.core.pab import pab_mgr as P
from videosys_b200.models.transformers.open_sora_transformer_3d import STDiT3, STDiT3Config

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
DEV = "cuda"


def _net(depth):
    cfg = dict(hidden_size=1152, num_heads=16, depth=depth, caption_channels=64, model_max_length=20)
    net = STDiT3(STDiT3Config(**cfg)).to(BF)
    net.load_state_dict(synth.fill_state_dict(net.state_dict(), "fp8gpu."))
    return net.to(DEV).eval()


def _inputs(T, H, W):
    inp = cases.forward_inputs(BF, T=T, H=H, W=W)
    return {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in inp.items()}


def _fwd(net, inp):
    with torch.no_grad():
        return net(inp["x"].to(BF), inp["timestep"].to(BF), inp["y"].to(BF), mask=inp["mask"], x_mask=inp["x_mask"],
                   fps=inp["fps"], height=inp["height"], width=inp["width"])


@pytest.mark.parametrize("grid", [(5, 12, 11), (4, 30, 53)], ids=["small", "240p"])
def test_fp8_forward_vs_bf16_and_toggle(grid):
    net = _net(depth=4)
    inp = _inputs(*grid)
    bf = _fwd(net, inp)
    net.set_fp8_linears(True)
    f8 = _fwd(net, inp)
    assert torch.equal(f8, _fwd(net, inp)), "FP8 forward is not deterministic"
    rel = ((f8.double() - bf.double()).norm() / bf.double().norm()).item()
    print(f"[fp8] grid {grid}: relative L2 of the FP8 velocity to the bf16 one {rel:.4e}")
    assert 0 < rel < 0.1
    net.set_fp8_linears(False)
    assert torch.equal(_fwd(net, inp), bf), "FP8 mode switched off does not reproduce the bf16 output"


def test_fp8_pab_step_graph_replay_bit_identical():
    net = _net(depth=2).set_fp8_linears(True)
    inp = _inputs(5, 12, 11)
    fwd = {k: v for k, v in inp.items() if k not in ("x", "timestep")}
    z0 = inp["x"][:1].to(BF).contiguous()
    ts = [torch.tensor([float(v)], device=DEV) for v in (1000, 900, 860, 800, 700, 600, 500, 300)]
    dts = [torch.tensor([0.05], device=DEV) for _ in ts]

    def run(graph):
        P.set_pab_manager(P.PABConfig(spatial_broadcast=True, spatial_threshold=[450, 930], spatial_range=2,
                                      temporal_broadcast=True, temporal_threshold=[450, 930], temporal_range=4,
                                      cross_broadcast=True, cross_threshold=[450, 930], cross_range=6))
        P.update_steps(len(ts))
        st = StepGraph(net, 7.0, enabled=graph)
        outs = []
        for _ in range(2):  # the second pass replays every skip pattern's graph
            net.reset_pab_state()
            z = z0.clone()
            for t, dt in zip(ts, dts):
                z = st.step(z, t, dt, fwd, ts_int=int(t.item()))
                outs.append(z.clone())
        return outs, st

    try:
        eager, _ = run(False)
        graphed, st = run(True)
    finally:
        P.set_pab_manager(None)
        net.reset_pab_state()
    assert st.replays >= len(ts), "the graph path was not taken"
    for i, (a, b) in enumerate(zip(eager, graphed)):
        assert torch.equal(a, b), f"step {i}: replayed FP8 graph differs from eager"
