"""OpenSora v1.2 conditioning: the helpers of pipelines/open_sora/conditioning.py against the reference's own functions
(executed unmodified, oracle/opensora_pipeline_ref.py) on a table of strategies, and ``generate`` with refs / ms / loop
around a stub denoiser, the native decoder and encoder on the kernel stand-ins: the encoded reference written into z,
the mask the sampler receives, the random draws in the reference's order, the loop's re-encode and time join, and each
rejection."""
import pytest
import torch

from oracle import ref_loader
from oracle.gen_golden_opensora_vae import NARROW, weights
from tests import kernels_emul_vae_down
from videosys_b200.models.autoencoders import OpenSoraVAEEncoder, VideoAutoencoderPipeline
from videosys_b200.pipelines.open_sora import conditioning as C


def _ref():
    if not ref_loader.available():
        pytest.skip("reference checkout not present")
    from oracle.opensora_pipeline_ref import load

    return load()


def _png(tmp_path, name="ref.png", size=(37, 23), seed=0):
    from PIL import Image

    g = torch.Generator().manual_seed(seed)
    arr = torch.randint(0, 256, (size[1], size[0], 3), generator=g, dtype=torch.uint8).numpy()
    p = tmp_path / name
    Image.fromarray(arr).save(p)
    return str(p)


# ---- the helpers against the reference ----
STRATEGIES = ["0", "0,0,0,0,1,0.5", "0,0,-1,-1,1,1.0", "0,0,0,3,2,0", "0,1,0,0,2;0,0,-2,-2,2,0.5", "1,0,0,0,1",
              "0,0,2,4,3,0.5", "0,1,-5,0,5,0.0;1,0,0,0,1", "0,0,1,7,4"]


@pytest.mark.parametrize("align", [None, 5, 2])
@pytest.mark.parametrize("ms", STRATEGIES)
def test_apply_mask_strategy_matches_reference(ms, align):
    P, _ = _ref()
    g = torch.Generator().manual_seed(1)
    refs = [[torch.randn(4, 6, 2, 3, generator=g), torch.randn(4, 9, 2, 3, generator=g)]]
    z0 = torch.randn(1, 4, 10, 2, 3, generator=g)
    for loop_i in (0, 1):
        za, zb = z0.clone(), z0.clone()
        ma = C.apply_mask_strategy(za, refs, [ms], loop_i, align=align)
        mb = P.apply_mask_strategy(zb, refs, [ms], loop_i, align=align)
        assert torch.equal(ma, mb) and torch.equal(za, zb)


def test_prompt_and_strategy_helpers_match_reference():
    P, _ = _ref()
    for s in ["", "0", "1,2", "0,1,-3,2,4,0.25;2,0", "0,0,0,0,1,1"]:
        assert C.parse_mask_strategy(s) == P.parse_mask_strategy(s)
    for args in [(0, 5, 10), (3, 5, 10), (8, 5, 10), (7, 5, 20), (13, 5, 15), (12, 5, 17), (4, 2, 9), (11, 4, 40)]:
        assert C.find_nearest_point(*args) == P.find_nearest_point(*args)
    for n in (5, 10, 20):
        assert C.dframe_to_frame(n) == P.dframe_to_frame(n)
    for p in ["a cat", "|0| a cat |2| a dog", "|0|sun|1|rain|3|snow"]:
        assert C.split_prompt(p) == P.split_prompt(p)
        merged = C.merge_prompt(*C.split_prompt(p))
        assert merged == P.merge_prompt(*P.split_prompt(p))
        for k in range(4):
            assert C.extract_prompts_loop([merged], k) == P.extract_prompts_loop([merged], k)
    for prompt in ["a cat", 'a cat{"reference_path": "x.png", "mask_strategy": "0"}', 'a dog{"mask_strategy": "0,0,0,0,2"}']:
        assert C.extract_json_from_prompts([prompt], ["r"], ["m"]) == P.extract_json_from_prompts([prompt], ["r"], ["m"])


@pytest.mark.parametrize("edit", [0.0, 0.5, 1.0])
def test_append_generated_matches_reference(edit):
    P, _ = _ref()
    lat = torch.randn(2, 4, 10, 2, 3)

    class _Vae:
        def encode(self, x):
            return lat

    for ms in (["", "0"], ["0,0,0,0,1", None]):
        ra, ma = C.append_generated(_Vae().encode, None, [[], [torch.zeros(1)]], list(ms), 1, 5, edit)
        rb, mb = P.append_generated(_Vae(), None, [[], [torch.zeros(1)]], list(ms), 1, 5, edit)
        assert ma == mb and all(len(a) == len(b) for a, b in zip(ra, rb))


@pytest.mark.parametrize("size", [(37, 23), (16, 64), (200, 100)])
def test_load_image_matches_reference(tmp_path, size):
    _, D = _ref()
    path = _png(tmp_path, size=size)
    for image_size in [(16, 24), (24, 16), (32, 32)]:
        want = D.read_from_path(path, image_size, transform_name="resize_crop")
        got = C.load_image(path, image_size)
        assert got.shape == want.shape == (3, 1, *image_size) and torch.equal(got, want)


def test_helper_rejections(tmp_path):
    with pytest.raises(ValueError, match="reference 1"):
        C.apply_mask_strategy(torch.zeros(1, 4, 5, 2, 3), [[torch.zeros(4, 1, 2, 3)]], ["0,1"], 0)
    with pytest.raises(ValueError, match="multiple of 5"):
        C.dframe_to_frame(3)
    with pytest.raises(ValueError, match="1 to 6"):
        C.parse_mask_strategy("0,0,0,0,1,0,7")
    with pytest.raises(ValueError, match="invalid key"):
        C.extract_json_from_prompts(['x{"seed": 1}'], [""], [""])
    with pytest.raises(NotImplementedError, match="video-file"):
        C.load_image(str(tmp_path / "clip.mp4"), (16, 24))
    with pytest.raises(ValueError, match="unsupported"):
        C.load_image(str(tmp_path / "a.txt"), (16, 24))


# ---- generate around a stub denoiser ----
class _RecordingScheduler:
    """Stands in for RFLOW.sample: records z (as the sampler receives it) and the mask, returns fixed latents."""

    def __init__(self):
        self.calls = []

    def sample(self, model, z, margs, y_null, dev, mask=None, progress=True):
        self.calls.append((z.clone(), None if mask is None else mask.clone()))
        g = torch.Generator().manual_seed(7 + len(self.calls))
        return torch.randn(z.shape, generator=g).to(z.dtype)


def _pipeline(monkeypatch, vae=True, encoder=True, **kw):
    from tests.test_opensora_vae_cpu import _StubTransformer
    from videosys_b200.pipelines.open_sora import pipeline_open_sora as P

    kernels_emul_vae_down.emulate(monkeypatch)
    monkeypatch.setitem(P._IMAGE_SIZE, ("144p", "9:16"), (16, 24))
    dec = enc = None
    if vae:
        dec = VideoAutoencoderPipeline(spatial_block_out_channels=NARROW).eval()
        dec.load_state_dict(weights(dec.state_dict(), "cond"))
    if encoder:
        enc = OpenSoraVAEEncoder(spatial_block_out_channels=NARROW).eval()
        enc.load_state_dict(weights(enc.state_dict(), "cond"))
    pipe = P.OpenSoraPipeline.__new__(P.OpenSoraPipeline)
    pipe._config = P.OpenSoraConfig(num_sampling_steps=2, **({} if dec is None else dict(vae=dec)),
                                    **({} if enc is None else dict(vae_encoder=enc)), **kw)
    pipe._device = torch.device("cpu")
    pipe.transformer = _StubTransformer()
    pipe.scheduler = _RecordingScheduler()
    pipe._set_seed = lambda seed: torch.manual_seed(seed)
    pipe.vae = pipe._load_vae()
    pipe._vae_encoder = None
    return pipe, enc


def _gen(pipe, **kw):
    kw = {"resolution": "144p", "aspect_ratio": "9:16", "num_frames": 17, "seed": 3, "verbose": False, **kw}
    return pipe.generate("a prompt", **kw).video


def test_generate_image_ref_writes_latent_and_mask_in_reference_order(monkeypatch, tmp_path):
    P, _ = _ref()
    pipe, enc = _pipeline(monkeypatch)
    png = _png(tmp_path)
    video = _gen(pipe, refs=png, ms="0")
    assert video.dtype == torch.uint8 and tuple(video.shape) == (1, 17, 16, 24, 3)
    (z, mask), = pipe.scheduler.calls
    # replay in the reference's order with its own helpers: seed, every reference encoded, z drawn, the strategy
    torch.manual_seed(3)

    class _Vae:
        device, dtype = torch.device("cpu"), torch.bfloat16

        def encode(self, x):
            return enc.encode(x)

    refs_x = P.collect_references_batch([png], _Vae(), (16, 24))
    z_ref = torch.randn(1, 4, 5, 2, 3, dtype=torch.bfloat16)
    masks = P.apply_mask_strategy(z_ref, refs_x, ["0"], 0, align=5)
    assert torch.equal(z, z_ref) and torch.equal(mask, masks)
    assert torch.equal(z[:, :, 0], refs_x[0][0][:, 0][None]) and mask.tolist() == [[0.0, 1.0, 1.0, 1.0, 1.0]]


def test_generate_loop2_reencodes_and_joins_along_time(monkeypatch, tmp_path):
    pipe, enc = _pipeline(monkeypatch)
    calls, outs = [], []
    orig = enc.encode
    monkeypatch.setattr(enc, "encode", lambda x: calls.append(x.clone()) or outs.append(orig(x)) or outs[-1])
    decoded = []
    orig_dec = pipe.vae.decode
    monkeypatch.setattr(pipe.vae, "decode", lambda z, num_frames=None: decoded.append(orig_dec(z, num_frames)) or decoded[-1].clone())
    video = _gen(pipe, num_frames=34, loop=2, refs=_png(tmp_path), ms="0")
    assert tuple(video.shape) == (1, 34 + (34 - 17), 16, 24, 3)  # nf + (loop - 1) * (nf - dframe_to_frame(5))
    assert len(calls) == 2 and torch.equal(calls[1], decoded[0])  # the decoded first clip is re-encoded
    (z0, m0), (z1, m1) = pipe.scheduler.calls
    assert m0[0, 0] == 0 and bool((m0[0, 1:] == 1).all())
    assert bool((m1[0, :5] == 0).all()) and bool((m1[0, 5:] == 1).all())  # "1,1,-5,0,5,0.0" on loop 1
    # the second clip's latent frames 0..4 are the last 5 latent frames of the re-encoded first clip
    assert outs[1].shape == (1, 4, 10, 2, 3) and torch.equal(z1[:, :, :5], outs[1][:, :, -5:])
    want = pipe._to_uint8(torch.cat([decoded[0], decoded[1][:, :, 17:]], dim=2))
    assert torch.equal(video, want)


def test_generate_loop_without_refs_appends_strategy(monkeypatch):
    pipe, _ = _pipeline(monkeypatch)
    video = _gen(pipe, num_frames=34, loop=3, condition_frame_edit=0.5)
    assert tuple(video.shape) == (1, 34 + 2 * 17, 16, 24, 3)
    masks = [m for _, m in pipe.scheduler.calls]
    assert bool((masks[0] == 1).all())
    for m in masks[1:]:
        assert bool((m[0, :5] == 0.5).all()) and bool((m[0, 5:] == 1).all())


def test_generate_conditioning_rejections(monkeypatch, tmp_path):
    png = _png(tmp_path)
    pipe, _ = _pipeline(monkeypatch, vae=False, encoder=False)
    for kw in (dict(refs=png, ms="0"), dict(loop=2), dict(ms="0")):
        with pytest.raises(ValueError, match="native OpenSora"):
            _gen(pipe, **kw)
    pipe, _ = _pipeline(monkeypatch, encoder=False)  # a decoder instance, no encoder to load
    with pytest.raises(ValueError, match="native OpenSora"):
        _gen(pipe, refs=png, ms="0")
    pipe, _ = _pipeline(monkeypatch)
    with pytest.raises(ValueError, match="reference 1"):
        _gen(pipe, refs=png, ms="0,1")
    with pytest.raises(ValueError, match="multiple of 5"):
        _gen(pipe, loop=2, condition_frame_length=3)
    with pytest.raises(NotImplementedError, match="video-file"):
        _gen(pipe, refs=str(tmp_path / "clip.mp4"), ms="0")
    pipe, _ = _pipeline(monkeypatch, vae_decode_fn=lambda s, nf: s)
    with pytest.raises(ValueError, match="vae_decode_fn"):
        _gen(pipe, refs=png, ms="0")


def test_generate_without_conditioning_unchanged(monkeypatch):
    """No refs / ms / loop: one sampler call with an all-ones mask, no encoder loaded, the plain decode."""
    pipe, _ = _pipeline(monkeypatch, encoder=False)
    video = _gen(pipe)
    (z, mask), = pipe.scheduler.calls
    assert pipe._vae_encoder is None and torch.equal(mask, torch.ones(1, 5))
    torch.manual_seed(3)
    assert torch.equal(z, torch.randn(1, 4, 5, 2, 3, dtype=torch.bfloat16))
    samples = torch.randn(z.shape, generator=torch.Generator().manual_seed(8)).to(z.dtype)
    assert torch.equal(video, pipe.decode_latents(samples, 17))
