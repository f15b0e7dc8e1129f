"""OpenSora v1.2 reference conditioning and looped generation: the helpers of the reference's generate()
(videosys/pipelines/open_sora/pipeline_open_sora.py: extract_json_from_prompts :719-733, collect_references_batch
:736-750, extract_prompts_loop :753-766, split_prompt :769-784, merge_prompt :787-794, MASK_DEFAULT / parse_mask_strategy
:797-815, find_nearest_point :818-822, apply_mask_strategy :825-854, append_generated :857-871, dframe_to_frame
:874-876) and the image loading of data_process.py (read_image_from_path :781-788 with the "resize_crop" transform
:712-719: pil_loader, resize_crop_to_fill :742-758, ToTensor, Normalize(0.5, 0.5)), restated.

Where the reference fails with an assertion or an IndexError on user input, these raise ValueError: a mask strategy
naming a reference that does not exist, more than six fields, a condition frame length that is not a multiple of 5, an
unsupported image extension, a JSON key other than reference_path / mask_strategy.  Video-file references raise
NotImplementedError: the reference's path hands the decoded frames (a tensor) to the PIL-only resize_crop_to_fill and
cannot run (data_process.py:742, ResizeCrop), and torchvision 0.26 has no read_video.
"""
import json
import os
import re

import numpy as np
import torch

VID_EXTENSIONS = (".mp4", ".avi", ".mov", ".mkv")  # data_process.py:26
IMG_EXTENSIONS = (".jpg", ".jpeg", ".png", ".ppm", ".bmp", ".pgm", ".tif", ".tiff", ".webp")  # torchvision's list
MASK_DEFAULT = ["0", "0", "0", "0", "1", "0"]  # loop id, ref id, ref start, target start, length, edit ratio


# ---- prompts ----
def extract_json_from_prompts(prompts, reference, mask_strategy):
    """A trailing JSON object in a prompt ({"reference_path": ..., "mask_strategy": ...}) overrides that sample's
    reference / mask strategy and is cut from the prompt."""
    out = []
    for i, prompt in enumerate(prompts):
        parts = re.split(r"(?=[{])", prompt)
        if len(parts) > 2:
            raise ValueError(f"invalid prompt (more than one JSON object): {prompt!r}")
        out.append(parts[0])
        if len(parts) > 1:
            for key, value in json.loads(parts[1]).items():
                if key == "reference_path":
                    reference[i] = value
                elif key == "mask_strategy":
                    mask_strategy[i] = value
                else:
                    raise ValueError(f"invalid key {key!r} in the prompt's JSON (reference_path, mask_strategy)")
    return out, reference, mask_strategy


def _loop_segments(prompt):
    """"|0|a|2|b" -> [(0, "a"), (2, "b")] (texts unstripped)."""
    parts = prompt.split("|")[1:]
    return [(int(parts[i]), parts[i + 1]) for i in range(0, len(parts), 2)]


def split_prompt(prompt_text):
    """A "|0| text |1| text ..." prompt -> (stripped texts, their first loops); any other prompt -> ([prompt], None)."""
    if not prompt_text.startswith("|0|"):
        return [prompt_text], None
    segs = _loop_segments(prompt_text)
    return [t.strip() for _, t in segs], [s for s, _ in segs]


def merge_prompt(text_list, loop_idx_list=None):
    if loop_idx_list is None:
        return text_list[0]
    return "".join(f"|{i}|{t}" for t, i in zip(text_list, loop_idx_list))


def extract_prompts_loop(prompts, num_loop):
    """Each prompt's text for loop ``num_loop``: a "|0|..." prompt's segment k covers loops start_k .. start_{k+1} - 1."""
    out = []
    for prompt in prompts:
        if prompt.startswith("|0|"):
            segs = _loop_segments(prompt)
            texts = []
            for k, (start, text) in enumerate(segs):
                end = segs[k + 1][0] if k + 1 < len(segs) else num_loop + 1
                texts.extend([text] * (end - start))
            prompt = texts[num_loop]
        out.append(prompt)
    return out


# ---- mask strategies ----
def parse_mask_strategy(mask_strategy):
    """"l,r,rs,ts,n,e;..." -> [[loop, ref, ref_start, target_start, length, edit_ratio], ...], missing trailing fields
    from MASK_DEFAULT."""
    if mask_strategy is None or mask_strategy == "":
        return []
    out = []
    for mask in mask_strategy.split(";"):
        group = mask.split(",")
        if not 1 <= len(group) <= 6:
            raise ValueError(f"invalid mask strategy {mask!r}: 1 to 6 comma-separated fields")
        group = group + MASK_DEFAULT[len(group):]
        out.append([int(v) for v in group[:5]] + [float(group[5])])
    return out


def find_nearest_point(value, point, max_value):
    """``value`` rounded to a multiple of ``point`` (down, or up past the half when that stays below the last multiple
    of ``point`` under ``max_value``)."""
    t = value // point
    if value % point > point / 2 and t < max_value // point - 1:
        t += 1
    return t * point


def apply_mask_strategy(z, refs_x, mask_strategys, loop_i, align=None):
    """Writes the referenced latent frames into z [B, C, T, h, w] in place and returns the per-frame mask [B, T]
    (float32 on z's device: 1 = generate, the strategy's edit ratio where a reference was written), None when there
    are no strategies at all."""
    if len(mask_strategys) == 0:
        return None
    masks = []
    for i, strategy in enumerate(mask_strategys):
        mask = torch.ones(z.shape[2], dtype=torch.float, device=z.device)
        for loop_id, m_id, ref_start, target_start, length, edit_ratio in parse_mask_strategy(strategy):
            if loop_id != loop_i:
                continue
            if not -len(refs_x[i]) <= m_id < len(refs_x[i]):
                raise ValueError(f"mask strategy {strategy!r} names reference {m_id}, but sample {i} has "
                                 f"{len(refs_x[i])} reference(s)")
            ref = refs_x[i][m_id]  # [C, T, h, w]
            if ref_start < 0:
                ref_start += ref.shape[1]
            if target_start < 0:
                target_start += z.shape[2]
            if align is not None:
                ref_start = find_nearest_point(ref_start, align, ref.shape[1])
                target_start = find_nearest_point(target_start, align, z.shape[2])
            length = min(length, z.shape[2] - target_start, ref.shape[1] - ref_start)
            z[i, :, target_start:target_start + length] = ref[:, ref_start:ref_start + length]
            mask[target_start:target_start + length] = edit_ratio
        masks.append(mask)
    return torch.stack(masks)


def dframe_to_frame(num):
    """Latent frames -> video frames of whole 17-frame micro batches (5 latent frames each)."""
    if num % 5 != 0:
        raise ValueError(f"condition_frame_length={num} must be a multiple of 5 (whole 17-frame VAE chunks)")
    return num // 5 * 17


def append_generated(encode, generated_video, refs_x, mask_strategy, loop_i, condition_frame_length,
                     condition_frame_edit):
    """Encodes the last clip ([B, 3, T, H, W]), appends each sample's latent to its references and a strategy that
    writes its last ``condition_frame_length`` latent frames to the front of loop ``loop_i``."""
    ref_x = encode(generated_video)
    for j, refs in enumerate(refs_x):
        refs.append(ref_x[j])
        mask_strategy[j] = "" if not mask_strategy[j] else mask_strategy[j] + ";"
        mask_strategy[j] += (f"{loop_i},{len(refs) - 1},-{condition_frame_length},0,{condition_frame_length},"
                             f"{condition_frame_edit}")
    return refs_x, mask_strategy


# ---- references ----
def resize_crop_to_fill(pil_image, image_size):
    """Bicubic resize so that the image covers (th, tw), then the centred crop (rounded offsets) on the long side."""
    from PIL import Image

    w, h = pil_image.size
    th, tw = image_size
    rh, rw = th / h, tw / w
    if rh > rw:
        sh, sw = th, round(w * rh)
        i, j = 0, int(round((sw - tw) / 2.0))
    else:
        sh, sw = round(h * rw), tw
        i, j = int(round((sh - th) / 2.0)), 0
    arr = np.array(pil_image.resize((sw, sh), Image.BICUBIC))
    return Image.fromarray(arr[i:i + th, j:j + tw])


def load_image(path, image_size):
    """An image file as a one-frame video [3, 1, H, W] in [-1, 1]: RGB, resize_crop_to_fill, ToTensor, Normalize(0.5,
    0.5)."""
    from PIL import Image

    ext = os.path.splitext(path)[-1].lower()
    if ext in VID_EXTENSIONS:
        raise NotImplementedError(f"{path}: video-file references are not supported (the reference's path passes the "
                                  "decoded frames to the PIL-only resize_crop_to_fill and cannot run); use an image")
    if ext not in IMG_EXTENSIONS:
        raise ValueError(f"{path}: unsupported image format {ext!r} (one of {IMG_EXTENSIONS})")
    with open(path, "rb") as f:
        img = Image.open(f).convert("RGB")
    img = resize_crop_to_fill(img, image_size)
    x = torch.from_numpy(np.array(img)).permute(2, 0, 1).contiguous().float().div(255)
    return x.sub_(0.5).div_(0.5)[:, None]


def collect_references_batch(reference_paths, encode, image_size):
    """Per sample the latents [C, T, h, w] of its ";"-separated reference files, each encoded on its own (every
    reference is encoded, used by a strategy or not, so the random draws stay in the reference's order)."""
    refs_x = []
    for reference_path in reference_paths:
        if reference_path == "":
            refs_x.append([])
            continue
        refs_x.append([encode(load_image(p, image_size)[None])[0] for p in reference_path.split(";")])
    return refs_x
