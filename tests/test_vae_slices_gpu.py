"""The VAE decoders and the OpenSora v1.2 encoder on the H100 under the sliced parity rule (tests/slice_parity.py): every
(sample, frame, 64 x 64 pixel tile) of the decoded video, and every (sample, frame) of the encoded latent, within the
eager 16-bit chain's own error of the fp32 chain, where the VAE tests elsewhere gate one relative L2 over a sample of the
whole output.

Each case decodes (or encodes) the same module and the same inputs three times: ``ours`` on the native kernels, ``r16``
on the kernels' torch stand-ins (tests/kernels_emul_vae*.py) in the same 16-bit dtype, and ``r32`` on the stand-ins with
the module in fp32 and TF32 off.  All three run the same front-end arithmetic, which the CPU and golden tests pin to the
reference; this file checks that the kernels are right in every frame and tile of it.  Each case crosses the seams of
its front end: CogVideoX's frame batches with carried conv caches and blended tiles, Open-Sora-Plan's time chunks (each
later one repeating the previous chunk's last frame) and blended tiles, OpenSora v1.2's 17-frame chunks with trimmed
padding and its image decoder's micro-batches of 4 frames, Latte's 14-frame chunks (the middle one straddling two
samples), Vchitect's 8-frame image-decoder passes.  The latents (and the encoder's video) are scaled and shifted frame by
frame, so that neighbouring frames differ in their statistics and a frame normalised with another's is visible.

The negative tests make one small in-bounds change to one kernel wrapper at one seam, or in one 64 x 64 region of the
final convolution, and require a worst slice at least NEGATIVE_MIN_LOAD times its bound, where correct code stays below
0.8.  Each prints whether the whole-output gate would have passed it.  The local tiles are asserted to pass that gate,
except at CogVideoX's 17 x 160 x 240 two-sample case: its fp16 error is small and one tile is 1/408 of the output, so the
whole-output gate fails that tile too; the same change at 49 x 480 x 720 passes it.

Scaling every down-sampling output of one image of the encoder by 1.05 moves the latent by less than the 16-bit error
(0.78 of the bound): each GroupNorm after it divides a uniform scaling of the image out, and four images fold into one
latent frame.  The encoder's micro-batch seam is checked by a GroupNorm statistics mix-up instead."""
import copy
import time

import pytest
import torch

from oracle.gen_golden_cogvideox_vae import CASES as COGX_CASES
from oracle.gen_golden_cogvideox_vae import weights as cogx_weights
from oracle.gen_golden_latte_vae import VCH_SCALE, VCH_SHIFT
from oracle.gen_golden_opensora_vae import RELEASED, weights
from oracle.gen_golden_osp_vae import V120_RELEASED
from oracle.gen_golden_osp_vae import weights as osp_weights
from tests import kernels_emul_vae as EV
from tests import kernels_emul_vae_down as ED
from tests import kernels_emul_vae_time as ET
from tests.slice_parity import assert_sliced_parity, sliced_parity
from videosys_b200 import kernels

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF, FP16 = torch.bfloat16, torch.float16
NEGATIVE_MIN_LOAD = 1.25


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _frame_varying(shape, seed, t_dim=2):
    """randn(shape), each frame (dimension t_dim) scaled by 1 + 0.3 sin(1.7 t) and shifted by 0.3 cos(2.3 t)."""
    x = torch.randn(shape, generator=torch.Generator().manual_seed(seed))
    t = torch.arange(shape[t_dim], dtype=torch.float32)
    view = [1] * len(shape)
    view[t_dim] = -1
    return x * (1 + 0.3 * torch.sin(1.7 * t)).view(view) + 0.3 * torch.cos(2.3 * t).view(view)


def _on_stand_ins(table, fn, fp32=False):
    with pytest.MonkeyPatch.context() as m:
        for n, f in table.items():
            m.setattr(kernels, n, f)
        if fp32:
            m.setattr(kernels, "require_cuda", lambda *a, **k: None)
            m.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
            m.setattr(torch.backends.cudnn, "allow_tf32", False)
        return fn()


# ---- the cases ---------------------------------------------------------------------------------------------------------
def _cogx(dtype, shape, tiled):
    cfg = COGX_CASES["released_f3"][0]
    from videosys_b200.models.autoencoders import AutoencoderKLCogVideoX

    vae = AutoencoderKLCogVideoX(**cfg)
    vae.load_state_dict(cogx_weights(vae.state_dict(), "released_f3"))
    vae = vae.to(dtype).to(DEV).eval()
    if tiled:
        vae.enable_tiling()
    return vae, _frame_varying(shape, 11), lambda m, z: m.decode(z).sample, EV.stand_ins(), "bcthw"


def _osp(version, dtype, shape):
    from videosys_b200.models.autoencoders.autoencoder_kl_open_sora_plan import decoder_class

    vae = decoder_class(version)(**(V120_RELEASED if version == "v120" else {}))
    vae.load_state_dict(osp_weights(vae.state_dict(), f"{version}_released"))
    vae = vae.to(dtype).to(DEV).eval()
    vae.enable_tiling()
    return vae, _frame_varying(shape, 12), lambda m, z: m.decode(z), EV.stand_ins(), "bcthw"


def _opensora_decoder():
    from videosys_b200.models.autoencoders import VideoAutoencoderPipeline

    vae = VideoAutoencoderPipeline(spatial_block_out_channels=RELEASED)
    vae.load_state_dict(weights(vae.state_dict(), "released"))
    vae = vae.to(BF).to(DEV).eval()
    return vae, _frame_varying((2, 4, 15, 30, 40), 13), lambda m, z: m.decode(z, num_frames=51), EV.stand_ins(), "bcthw"


def _zero_noise_encode(m, x):
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(torch, "randn", lambda *s, **kw: torch.zeros(*s, **{k: v for k, v in kw.items() if k != "generator"}))
        return m.encode(x)


def _opensora_encoder():
    from videosys_b200.models.autoencoders import OpenSoraVAEEncoder

    enc = OpenSoraVAEEncoder(spatial_block_out_channels=RELEASED)
    enc.load_state_dict(weights(enc.state_dict(), "released"))
    enc = enc.to(BF).to(DEV).eval()
    x = (_frame_varying((2, 3, 51, 240, 320), 14) / 2.5).clamp(-1, 1)
    return enc, x, _zero_noise_encode, ED.stand_ins(), "bcthw"


def _latte():
    from videosys_b200.models.autoencoders import AutoencoderKLTemporalDecoder
    from videosys_b200.pipelines.latte import pipeline_latte as P

    vae = AutoencoderKLTemporalDecoder(block_out_channels=RELEASED)
    vae.load_state_dict(weights(vae.state_dict(), "latte/real"))
    vae = vae.to(FP16).to(DEV).eval()

    def decode(m, z):
        pipe = P.LattePipeline.__new__(P.LattePipeline)
        pipe._config, pipe._device, pipe._dtype, pipe.vae = P.LatteConfig(vae=m), torch.device(DEV), torch.float16, m
        return pipe.decode_video(z)

    return vae, _frame_varying((2, 4, 16, 64, 64), 15), decode, ET.stand_ins(), "bthwc"


def _vchitect():
    from videosys_b200.models.autoencoders import AutoencoderKL
    from videosys_b200.pipelines._common import decode_image_frames

    vae = AutoencoderKL(block_out_channels=RELEASED, latent_channels=16, use_post_quant_conv=False, scaling_factor=VCH_SCALE,
                        shift_factor=VCH_SHIFT)
    vae.load_state_dict(weights(vae.state_dict(), "vchitect/released"))
    vae = vae.to(BF).to(DEV).eval()

    def decode(m, z):  # the pipeline's decode tail: 40 frames of 288 x 480, VAE_FRAMES_PER_PASS = 8 frames per pass
        return decode_image_frames(m, ((z / m.config.scaling_factor) + m.config.shift_factor)[0])

    return vae, _frame_varying((1, 40, 16, 36, 60), 16, t_dim=1), decode, ET.stand_ins(), "tchw"


# name: (builder, what the case crosses)
CASES = {
    "cogvideox_tiled_fp16": (lambda: _cogx(FP16, (1, 16, 13, 60, 90), True),
                             "49 x 480 x 720; frame batches 3+2+2+2+2+2 with carried caches; 3 x 3 blended tiles"),
    "cogvideox_b2_bf16": (lambda: _cogx(BF, (2, 16, 5, 20, 30), False), "frame batches 3+2; two samples"),
    "cogvideox_b2_fp16": (lambda: _cogx(FP16, (2, 16, 5, 20, 30), False), "frame batches 3+2; two samples"),
    "osp_v120_bf16": (lambda: _osp("v120", BF, (1, 4, 17, 36, 36)),
                      "latent time chunks [0, 16) [15, 17), the repeated frame dropped; 2 x 2 blended tiles"),
    "osp_v110_fp16": (lambda: _osp("v110", FP16, (1, 4, 18, 36, 36)),
                      "latent time chunks [0, 17) [16, 18) with TimeUpsample2x; 2 x 2 blended tiles"),
    "opensora_decoder_bf16": (_opensora_decoder, "51 frames of 240 x 320: 3 chunks with trimmed padding; image micro-batches "
                                                 "of 4 ending in a partial one; two samples"),
    "opensora_encoder_bf16": (_opensora_encoder, "51 frames of 240 x 320 in: image micro-batches of 4, 3 chunks of 17 frames; "
                                                 "two samples; posterior mode"),
    "latte_fp16": (_latte, "2 x 16 frames of 512 x 512: chunks 14, 14, 4, the middle one straddling the samples"),
    "vchitect_bf16": (_vchitect, "40 frames of 288 x 480 in 5 passes of 8"),
}


def _build(name):
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    module, x32, run, table, axes = CASES[name][0]()
    x = x32.to(module.dtype if hasattr(module, "dtype") else BF).to(DEV)
    n0 = kernels.launch_count()
    ours = run(module, x)
    launches = kernels.launch_count() - n0
    assert launches > 50, f"{name}: only {launches} native launches"
    assert torch.equal(ours, run(module, x)), f"{name}: two native runs differ"
    r16 = _on_stand_ins(table, lambda: run(module, x))
    m32 = copy.deepcopy(module).float()
    r32 = _on_stand_ins(table, lambda: run(m32, x.float()), fp32=True)
    del m32
    torch.cuda.synchronize()
    c = dict(module=module, x=x, run=run, axes=axes, ours=ours, r16=r16, r32=r32, launches=launches,
             seconds=time.perf_counter() - t0, peak=torch.cuda.max_memory_allocated())
    torch.cuda.empty_cache()
    return c


@pytest.fixture(scope="module")
def vae_case():
    """case(name) -> the module, its input and its three outputs, built once per module."""
    store = {}

    def get(name):
        if name not in store:
            store[name] = _build(name)
        return store[name]

    yield get
    store.clear()
    torch.cuda.empty_cache()


@pytest.mark.parametrize("name", list(CASES))
def test_vae_sliced(vae_case, name):
    _need_gpu()
    c = vae_case(name)
    print(f"[vae slices] {name}: {CASES[name][1]}; output {tuple(c['ours'].shape)}; {c['launches']} native launches; "
          f"three runs + the rule {c['seconds']:.1f} s, peak device memory {c['peak'] / 2**30:.1f} GiB")
    assert_sliced_parity(f"vae {name}", c["ours"], c["r16"], c["r32"], c["axes"])


# ---- negative tests: one small in-bounds change to one kernel wrapper -----------------------------------------------------
def _counting(mp, obj, attr, state):
    """obj.attr counts its calls in state["n"] (the frame batch, chunk or micro-batch being run)."""
    f = getattr(obj, attr)

    def counted(*a, **kw):
        state["n"] += 1
        return f(*a, **kw)

    mp.setattr(obj, attr, counted)


def _cogx_seam(mp, vae):
    """The second frame batch's conv_in reads zero context frames: the conv cache is not carried into it."""
    state, f = {"n": 0, "done": False}, kernels.vae_conv3d
    _counting(mp, vae.decoder, "forward", state)

    def vae_conv3d(x, *a, **kw):
        if state["n"] == 2 and not state["done"]:
            state["done"] = True
            x = x.clone()
            x[:, :2] = 0
        return f(x, *a, **kw)

    mp.setattr(kernels, "vae_conv3d", vae_conv3d)


def _opensora_neighbour_stats(mp, vae):
    """In the image decoder's fourth micro-batch (frames 12-15 of sample 0), frame 13 is normalised with frame 12's
    GroupNorm statistics, in every GroupNorm."""
    state, f = {"n": 0}, kernels.vae_groupnorm_stats
    _counting(mp, vae.spatial_vae.module, "decode_frames", state)

    def vae_groupnorm_stats(x, *a, **kw):
        s = f(x, *a, **kw)
        if state["n"] == 4:
            s = s.clone()
            s[1] = s[0]
        return s

    mp.setattr(kernels, "vae_groupnorm_stats", vae_groupnorm_stats)


def _latte_straddle_mix(mp, vae):
    """In the middle chunk (flattened frames 14-27: sample 0's last two, sample 1's first twelve), frame 2 of the chunk
    (sample 1, frame 0) takes the AlphaBlender's temporal weight x 1.02 in every temporal resnet."""
    state, f = {"n": 0}, kernels.vae_conv_time
    _counting(mp, vae, "decode", state)

    def vae_conv_time(x, w, b, cout, kt, resid=None, mix=None, **kw):
        out = f(x, w, b, cout, kt, resid=resid, mix=mix, **kw)
        if state["n"] == 2 and mix is not None:
            out[:, 2] = f(x, w, b, cout, kt, resid=resid, mix=(mix[0], 1.02 * mix[1]), **kw)[:, 2]
        return out

    mp.setattr(kernels, "vae_conv_time", vae_conv_time)


def _osp_second_chunk_upsample(mp, vae):
    """In the second time chunk, the first frame of every vae_upsample_linear2x output x 1.05."""
    state, f = {"n": 0}, kernels.vae_upsample_linear2x
    _counting(mp, vae, "tiled_decode2d", state)

    def vae_upsample_linear2x(x, spatial, temporal, out=None, t_off=0):
        y = f(x, spatial, temporal, out=out, t_off=t_off)
        if state["n"] == 2:
            y[:, t_off if out is not None else 0].mul_(1.05)
        return y

    mp.setattr(kernels, "vae_upsample_linear2x", vae_upsample_linear2x)


def _encoder_neighbour_stats(mp, enc):
    """In the image encoder's fourth micro-batch, its second image is normalised with the first one's GroupNorm
    statistics, in every GroupNorm."""
    state, f = {"n": 0}, kernels.vae_groupnorm_stats
    _counting(mp, enc.spatial_vae.module, "moments", state)

    def vae_groupnorm_stats(x, *a, **kw):
        s = f(x, *a, **kw)
        if state["n"] == 4:
            s = s.clone()
            s[1] = s[0]
        return s

    mp.setattr(kernels, "vae_groupnorm_stats", vae_groupnorm_stats)


def _local_tile(entry):
    """The first call of the final RGB convolution (``entry``) writes x 1.05 into rows and columns 64-127 of the first
    frame of its first sample: one 64 x 64 tile of one frame of the output."""

    def patch(mp, vae):
        state, f = {"done": False}, getattr(kernels, entry)

        def final(*a, **kw):
            y = f(*a, **kw)
            if y.shape[-1] == 3 and not state["done"]:
                state["done"] = True
                y[0, 0, 64:128, 64:128].mul_(1.05)
            return y

        mp.setattr(kernels, entry, final)

    return patch


# id: (case, change, patch, whether the whole-output gate is expected to pass it)
NEGATIVE = {
    "cogx_seam": ("cogvideox_b2_fp16", "second frame batch's conv_in without the carried cache", _cogx_seam, False),
    "opensora_stats": ("opensora_decoder_bf16", "image micro-batch frame normalised with its neighbour's statistics",
                       _opensora_neighbour_stats, False),
    "latte_straddle": ("latte_fp16", "straddling chunk, one frame's temporal mix weight x 1.02", _latte_straddle_mix, False),
    "osp_chunk": ("osp_v120_bf16", "second time chunk, first up-sampled frame x 1.05", _osp_second_chunk_upsample, False),
    "encoder_stats": ("opensora_encoder_bf16", "image micro-batch image normalised with its neighbour's statistics",
                      _encoder_neighbour_stats, False),
    "cogx_tile": ("cogvideox_b2_fp16", "conv_out x 1.05 in one 64 x 64 tile", _local_tile("vae_conv3d"), False),
    "cogx_tiled_tile": ("cogvideox_tiled_fp16", "conv_out x 1.05 in one 64 x 64 tile", _local_tile("vae_conv3d"), True),
    "osp_tile": ("osp_v120_bf16", "conv_out x 1.05 in one 64 x 64 tile", _local_tile("vae_conv3d"), True),
    "opensora_tile": ("opensora_decoder_bf16", "conv_out x 1.05 in one 64 x 64 tile", _local_tile("vae_conv3d"), True),
    "latte_tile": ("latte_fp16", "time_conv_out x 1.05 in one 64 x 64 tile", _local_tile("vae_time_conv_rgb"), True),
    "vchitect_tile": ("vchitect_bf16", "conv_out x 1.05 in one 64 x 64 tile", _local_tile("vae_conv3d"), True),
}


@pytest.mark.parametrize("neg", list(NEGATIVE))
def test_vae_negative_rejected(vae_case, neg):
    _need_gpu()
    name, change, patch, below_old_gate = NEGATIVE[neg]
    c = vae_case(name)
    with pytest.MonkeyPatch.context() as mp:
        patch(mp, c["module"])
        got = c["run"](c["module"], c["x"])
    rep = sliced_parity(f"NEGATIVE vae {name}: {change}", got, c["r16"], c["r32"], c["axes"])
    print(rep.describe())
    assert rep.worst >= NEGATIVE_MIN_LOAD, f"{change}: worst slice only {rep.worst:.3f}x its bound"
    if below_old_gate:
        assert rep.old_gate_ok, f"{change}: meant as a change the whole-output gate does not see ({rep.whole_ratio:.3f})"
