"""Parity of the CUDA image transform (csrc/preprocess.cu, through the C ABI) with the oracle and with
the reference's own test_tensors goldens: bit-exact float32."""
import hashlib
import os

import numpy as np
import pytest
import torch

import clip_retrieval_b200 as b200
from oracle import preprocess_ref as P

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "preprocess_ref.npz")


def _rand(shape, seed):
    return np.random.default_rng(seed).integers(0, 256, (*shape, 3), dtype=np.uint8)


def test_reference_goldens_bit_exact():
    g = np.load(GOLD)
    names = [n for n in g["names"] if f"pixels_{n}" in g.files]
    pre = b200.B200Preprocess(224)
    out = pre([g[f"pixels_{n}"] for n in names]).cpu().numpy()
    for i, n in enumerate(names):
        assert hashlib.sha256(np.ascontiguousarray(out[i]).tobytes()).digest() == g[f"sha256_{n}"].tobytes(), n
        assert np.array_equal(out[i], P.preprocess(g[f"pixels_{n}"]))


@pytest.mark.parametrize("n_px", [224, 336])
def test_ragged_batch_matches_oracle(n_px):
    shapes = [(224, 224), (300, 224), (224, 301), (375, 500), (500, 375), (225, 226), (97, 64), (1, 1), (3, 700),
              (1333, 800), (449, 448), (n_px, n_px), (n_px, 2 * n_px), (2000, 3000), (37, 4100)]
    imgs = [_rand(s, 100 + i) for i, s in enumerate(shapes)]
    pre = b200.B200Preprocess(n_px)
    out = pre(imgs).cpu().numpy()
    assert out.shape == (len(imgs), 3, n_px, n_px) and out.dtype == np.float32
    for i, im in enumerate(imgs):
        want = P.preprocess(im, n_px)
        assert np.array_equal(out[i], want), (shapes[i], float(np.abs(out[i] - want).max()))


def test_constant_and_extreme_pixels():
    imgs = [np.zeros((300, 500, 3), np.uint8), np.full((500, 300, 3), 255, np.uint8),
            np.tile(np.array([[[0, 255, 0]], [[255, 0, 255]]], np.uint8), (150, 400, 1))]
    out = b200.B200Preprocess(224)(imgs).cpu().numpy()
    for i, im in enumerate(imgs):
        assert np.array_equal(out[i], P.preprocess(im))


def test_device_pixels_and_reuse():
    pre = b200.B200Preprocess(224)
    imgs = [_rand((256, 320), 1), _rand((640, 480), 2)]
    buf, off, hh, ww = pre.pack(imgs)
    host = pre.run_packed(buf, off, hh, ww).cpu().numpy()
    dev = pre.run_packed(torch.from_numpy(buf).cuda(), off, hh, ww).cpu().numpy()
    assert np.array_equal(host, dev)
    small = pre([_rand((230, 230), 3)]).cpu().numpy()          # shrinking batch reuses the workspaces
    assert np.array_equal(small[0], P.preprocess(_rand((230, 230), 3)))
    assert pre([]).shape == (0, 3, 224, 224)


def test_bad_arguments_raise():
    pre = b200.B200Preprocess(224)
    with pytest.raises(ValueError):
        pre([np.zeros((4, 4, 4), np.uint8)])
    with pytest.raises(b200.B200Error):
        pre.run_packed(np.zeros(12, np.uint8), [0], [0], [4])


def test_mapper_accepts_raw_images():
    mapper = b200.ClipMapper(True, False, False, False, "synthetic:ViT-B/32", False, "", warmup_batch_size=4)
    n_px = mapper.model.arch.image_size
    imgs = [_rand((n_px + 40, n_px + 13), 11), _rand((n_px * 2, n_px * 3), 12), _rand((n_px, n_px), 13)]
    via_gpu = mapper({"image_rgb8": imgs, "image_filename": ["a", "b", "c"]})["image_embs"]
    tens = torch.from_numpy(P.preprocess_batch(imgs, n_px))
    via_host = mapper({"image_tensor": tens, "image_filename": ["a", "b", "c"]})["image_embs"]
    assert via_gpu.dtype == np.float16 and via_gpu.shape == via_host.shape
    assert np.array_equal(via_gpu, via_host)


@pytest.mark.timeout(300)
def test_gpu_jpeg_decode_feeds_the_transform():
    """nvJPEG decode in front of the GPU transform (the reference decodes with PIL on the host, reader.py:98-106).
    JPEG decoders are not bit-identical (IDCT rounding, chroma upsampling): bounded in grey levels against the
    Pillow-decoded pixels of the same files, and in cosine on what the image tower makes of them."""
    import torch
    import clip_retrieval_b200 as m
    from oracle import clip_ref

    here = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    gold = np.load(os.path.join(here, "jpeg_pixels.npz"))
    names = ["a_444", "b_420", "c_gray"]
    blobs = [open(os.path.join(here, "jpeg", n + ".jpg"), "rb").read() for n in names]
    pre = m.B200Preprocess(224)
    for n, blob in zip(names, blobs):
        got = pre.decode_jpeg_bytes(blob)
        want = gold[n]
        assert got.shape == want.shape and got.dtype == np.uint8
        diff = np.abs(got.astype(np.int32) - want.astype(np.int32))
        # nvJPEG and Pillow upsample chroma differently (4:2:0): bounds on the mean and 99th percentile, not bit-exactness
        assert diff.mean() <= 2.5 and np.percentile(diff, 99) <= 10, (n, diff.mean(), np.percentile(diff, 99), diff.max())
    # the batch path: decode + transform on the device, plus one non-JPEG blob that must fall back to the host decode
    import io
    from PIL import Image

    png = io.BytesIO()
    Image.fromarray(gold["a_444"]).save(png, format="PNG")
    batch = pre.from_jpeg_bytes(blobs + [png.getvalue()])
    ref = pre([gold[n] for n in names] + [gold["a_444"]])           # transform of the Pillow-decoded pixels
    assert batch.shape == ref.shape == (4, 3, 224, 224)
    assert torch.equal(batch[3], ref[3])                             # host-decoded fallback: identical pixels
    assert float((batch[:3] - ref[:3]).abs().mean()) <= 0.03         # in units of the normalised tensor (1 level ~ 0.015)
    cfg = clip_ref.CONFIGS["ViT-B/32"]
    model = m.B200Clip(m.ARCHS["ViT-B/32"], device=0, max_batch=4).load_state_dict(clip_ref.make_state_dict(cfg, seed=0))
    ea, eb = model.embed_image_device(batch), model.embed_image_device(ref)
    cos = torch.nn.functional.cosine_similarity(ea.float(), eb.float(), dim=-1)
    assert float(cos.min()) >= 0.999, cos
