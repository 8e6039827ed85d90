"""The squash transform of open_clip's `resize_mode="squash"` on the CPU: bicubic `Resize((n_px, n_px))` with no centre
crop, then ToTensor and Normalize.  It reuses the Pillow-exact resampler of oracle/preprocess_ref.py (pinned there
against Pillow + torchvision and the reference's fixtures) and only changes the output size: both sides go to n_px
whatever the aspect ratio.  tests/test_h14_378_cpu.py pins it against Pillow's `Image.resize((n, n), BICUBIC)`."""
import numpy as np

from oracle import preprocess_ref as P


def preprocess_squash(img_u8, n_px, mean=P.OPENAI_MEAN, std=P.OPENAI_STD):
    """uint8 RGB [H,W,3] -> float32 [3,n_px,n_px]."""
    img_u8 = np.ascontiguousarray(img_u8)
    assert img_u8.dtype == np.uint8 and img_u8.ndim == 3 and img_u8.shape[2] == 3
    if img_u8.shape[:2] != (n_px, n_px):              # torchvision short-circuits an already-sized image
        img_u8 = P.resize_bicubic(img_u8, n_px, n_px)
    x = img_u8.astype(np.float32) / np.float32(255)
    x = (x - np.asarray(mean, np.float32)) / np.asarray(std, np.float32)
    return np.ascontiguousarray(x.transpose(2, 0, 1))


def preprocess_squash_batch(images, n_px):
    return np.stack([preprocess_squash(im, n_px) for im in images])


def preprocess(img_u8, n_px, resize_mode):
    """The host transform of either resize mode: "shortest" is oracle/preprocess_ref.py's, "squash" the one above."""
    assert resize_mode in ("shortest", "squash"), resize_mode
    return preprocess_squash(img_u8, n_px) if resize_mode == "squash" else P.preprocess(img_u8, n_px)
