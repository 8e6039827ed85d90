"""ViT-H/14 at 378 px (`open_clip:ViT-H-14-378-quickgelu`, DFN5B): T = 730 image tokens at head dim 80, which only
the streaming attention kernel runs.  The real-size synthetic tower against the fp32 oracle, the mapper on
`image_tensor` and on `image_rgb8` through the squash transform, and batch-1 graph replay against eager launches."""
import os

import numpy as np
import pytest

from oracle import clip_ref
import squash_ref as S

pytestmark = pytest.mark.gpu
COS_TOL = 1e-3
NAME = "synthetic:open_clip:ViT-H-14-378-quickgelu"
CFG = clip_ref.ClipCfg(1024, 378, 14, clip_ref.TowerCfg(1280, 32, 16, 5120), clip_ref.TowerCfg(1024, 24, 16, 4096),
                       quick_gelu=True, name="ViT-H-14-378")


def _rand(shape, seed):
    return np.random.default_rng(seed).integers(0, 256, (*shape, 3), dtype=np.uint8)


@pytest.fixture(scope="module")
def model_and_sd():
    import clip_retrieval_b200 as m

    sd = clip_ref.make_state_dict(CFG, seed=0)
    arch, _ = m.model.resolve_arch(NAME)
    assert (arch.image_size // arch.patch) ** 2 + 1 == 730 and arch.quick_gelu
    model = m.B200Clip(arch, device=0, max_batch=2).load_state_dict(sd)
    return model, sd


@pytest.mark.timeout(1200)
def test_tower_matches_oracle(model_and_sd):
    import torch

    torch.set_num_threads(max(1, os.cpu_count() or 1))
    model, sd = model_and_sd
    px = clip_ref.synth_images(2, CFG, seed=1)
    tk = clip_ref.synth_tokens(2, CFG, seed=1)
    fi = model.encode_image(px.cuda()).cpu().numpy()
    ref_i = clip_ref.encode_image(sd, CFG, px).numpy()
    assert (1 - clip_ref.cosine(fi, ref_i)).max() <= COS_TOL, 1 - clip_ref.cosine(fi, ref_i)
    np.testing.assert_allclose(np.linalg.norm(fi, axis=1), np.linalg.norm(ref_i, axis=1), rtol=2e-2)
    ei, et = model.embed_image(px), model.embed_text(tk)
    ci = 1 - clip_ref.cosine(ei, clip_ref.mapper_image(sd, CFG, px))
    ct = 1 - clip_ref.cosine(et, clip_ref.mapper_text(sd, CFG, tk))
    assert ci.max() <= COS_TOL and ct.max() <= COS_TOL, (ci, ct)
    # device path == host path bit for bit
    assert np.array_equal(model.embed_image_device(px.cuda()).cpu().numpy(), ei)


@pytest.mark.timeout(600)
def test_batch1_graph_replay_equals_eager(model_and_sd):
    """Call 0 runs eagerly, call 1 captures the batch-1 graph, calls 2.. replay it: all equal bit for bit."""
    import torch

    model, _ = model_and_sd
    px = clip_ref.synth_images(1, CFG, seed=5).cuda()
    outs = [model.encode_image(px) for _ in range(4)]
    for o in outs[1:]:
        assert torch.equal(o, outs[0])


@pytest.mark.timeout(900)
def test_mapper_image_tensor_and_squashed_rgb8():
    import torch
    import clip_retrieval_b200 as b200

    n_px = 378
    imgs = [_rand((n_px + 40, n_px + 13), 11), _rand((200, 640), 12), _rand((n_px, n_px), 13)]
    # the GPU squash transform equals the oracle's pixels bit for bit
    squash = S.preprocess_squash_batch(imgs, n_px)
    got = b200.B200Preprocess(n_px, resize_mode="squash")(imgs).cpu().numpy()
    assert np.array_equal(got, squash)

    mapper = b200.ClipMapper(True, False, False, False, NAME + "/dfn5b", False, "", warmup_batch_size=3)
    assert mapper.model.arch.image_size == n_px
    tens = torch.from_numpy(squash)
    via_host = mapper({"image_tensor": tens, "image_filename": ["a", "b", "c"]})["image_embs"]
    assert via_host.dtype == np.float16 and via_host.shape == (3, 1024)
    np.testing.assert_allclose(np.linalg.norm(via_host.astype(np.float32), axis=1), 1.0, atol=2e-3)
    via_dev = mapper.model.embed_image_device(tens.cuda()).cpu().numpy()
    assert np.array_equal(via_dev, via_host)
    via_rgb8 = mapper({"image_rgb8": imgs, "image_filename": ["a", "b", "c"]})["image_embs"]
    assert np.array_equal(via_rgb8, via_host)
