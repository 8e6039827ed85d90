"""`open_clip:ViT-H-14-378-quickgelu` (DFN5B) without a GPU: how its names resolve, the squash transform's CPU
restatement (squash_ref.py) against Pillow + torchvision, and which names get that transform."""
import os

import numpy as np
import pytest

import squash_ref as S
from oracle import preprocess_ref as P

REF_IMAGES = os.path.join(os.path.dirname(__file__), "golden", "ref_images")


@pytest.mark.parametrize("name,quick", [
    ("open_clip:ViT-H-14-378", False),
    ("open_clip:ViT-H-14-378-quickgelu", True),
    ("open_clip:ViT-H-14-378-quickgelu/dfn5b", True),
    ("synthetic:open_clip:ViT-H-14-378-quickgelu", True),
])
def test_resolve_arch(name, quick):
    from clip_retrieval_b200.model import _find_checkpoint, resolve_arch

    arch, key = resolve_arch(name)
    assert arch.vision.width == 1280 and arch.vision.layers == 32 and arch.vision.heads == 16
    assert arch.text.width == 1024 and arch.embed_dim == 1024
    assert (arch.image_size // arch.patch) ** 2 + 1 == 730
    assert arch.vision.width // arch.vision.heads == 80
    assert arch.quick_gelu == quick
    assert key == "open_clip:ViT-H-14-378" + ("-quickgelu" if quick else "")
    assert _find_checkpoint(key, None) is None


def test_checkpoint_stem(tmp_path):
    from clip_retrieval_b200.model import _find_checkpoint, resolve_arch

    _, key = resolve_arch("open_clip:ViT-H-14-378-quickgelu/dfn5b")
    p = tmp_path / "ViT-H-14-378-quickgelu.pt"
    p.write_bytes(b"")
    assert _find_checkpoint(key, str(tmp_path)) == str(p)


def _squash_torchvision(n_px):
    from torchvision import transforms as T
    from torchvision.transforms import InterpolationMode

    return T.Compose([T.Resize((n_px, n_px), interpolation=InterpolationMode.BICUBIC),
                      lambda im: im.convert("RGB"), T.ToTensor(), T.Normalize(P.OPENAI_MEAN, P.OPENAI_STD)])


def test_oracle_squash_matches_pillow_on_ref_images():
    from PIL import Image

    names = sorted(os.listdir(REF_IMAGES))
    assert len(names) == 7
    for n_px in (224, 378):
        for name in names:
            im = Image.open(os.path.join(REF_IMAGES, name)).convert("RGB")
            # Image.resize((n, n), BICUBIC) -> ToTensor -> Normalize
            ref = _squash_torchvision(n_px)(im).numpy()
            direct = np.asarray(im.resize((n_px, n_px), Image.BICUBIC), np.float32) / np.float32(255)
            direct = ((direct - np.asarray(P.OPENAI_MEAN, np.float32)) / np.asarray(P.OPENAI_STD, np.float32))
            got = S.preprocess_squash(np.asarray(im), n_px)
            assert got.shape == (3, n_px, n_px)
            assert np.array_equal(got, ref), (name, n_px)
            assert np.array_equal(got, direct.transpose(2, 0, 1)), (name, n_px)


@pytest.mark.parametrize("shape", [(378, 378), (200, 640), (700, 301), (1, 1)])
def test_oracle_squash_synthetic_shapes(shape):
    from PIL import Image

    px = np.random.default_rng(shape[0] * 31 + shape[1]).integers(0, 256, (*shape, 3), dtype=np.uint8)
    assert np.array_equal(S.preprocess_squash(px, 378), _squash_torchvision(378)(Image.fromarray(px)).numpy())


@pytest.mark.parametrize("name,mode", [
    ("open_clip:ViT-H-14-378-quickgelu/dfn5b", "squash"),
    ("open_clip:ViT-H-14-378/dfn5b", "squash"),
    ("synthetic:open_clip:ViT-H-14-378-quickgelu/dfn5b", "squash"),
    ("open_clip:ViT-H-14-378-quickgelu", "shortest"),
    ("synthetic:open_clip:ViT-H-14-378-quickgelu", "shortest"),
    ("open_clip:ViT-H-14-quickgelu/dfn5b", "shortest"),      # the 224-px DFN5B tower keeps today's transform
    ("open_clip:ViT-H-14/laion2b_s32b_b79k", "shortest"),
    ("ViT-L/14", "shortest"),
])
def test_transform_choice(name, mode):
    from PIL import Image

    from clip_retrieval_b200.model import make_preprocess, preprocess_mode, resolve_arch

    assert preprocess_mode(name) == mode
    n_px = resolve_arch(name)[0].image_size
    px = np.random.default_rng(3).integers(0, 256, (n_px + 50, n_px + 7, 3), dtype=np.uint8)
    got = make_preprocess(n_px, preprocess_mode(name))(Image.fromarray(px)).numpy()
    assert np.array_equal(got, S.preprocess(px, n_px, mode))
