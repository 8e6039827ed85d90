"""GPU image transform (SURVEY §8(f) row 1): the `preprocess` step of the reference's readers
(clip_retrieval/clip_inference/reader.py:98-106,158-165) moved behind the C ABI.

`B200Preprocess(n_px)(images)` takes decoded images (PIL.Image or uint8 HWC arrays, any sizes) and
returns the float32 `[n, 3, n_px, n_px]` batch on the device that `ClipMapper` / `encode_image`
consume — bit-identical to torchvision's Compose[Resize(bicubic), CenterCrop, ToTensor, Normalize]
on the host (tests/test_preprocess_gpu.py; pinned on the reference's own test_tensors fixtures).
`resize_mode="squash"` resizes both sides to n_px with no crop instead (Resize((n_px, n_px)), open_clip's
"squash"), the transform of the checkpoints that `model.preprocess_mode` names.
`B200Preprocess.from_jpeg_bytes(list_of_bytes)` additionally decodes on the GPU (nvJPEG): what crosses PCIe is the
compressed file.  Streams nvJPEG cannot parse fall back to PIL on the host, as the reference decodes every image."""
import ctypes as C

import numpy as np
import torch

from ._lib import lib, check

OPENAI_MEAN = (0.48145466, 0.4578275, 0.40821073)
OPENAI_STD = (0.26862954, 0.26130258, 0.27577711)
RESIZE_MODES = {"shortest": 0, "squash": 1}   # B200_RESIZE_SHORTEST / B200_RESIZE_SQUASH


def to_rgb8(image):
    """PIL.Image | ndarray -> contiguous uint8 [H, W, 3].  Mode conversion happens before the resize
    (the reference converts after it; identical for RGB and L sources, which is what JPEG yields)."""
    if isinstance(image, np.ndarray):
        a = image
    else:
        a = np.asarray(image.convert("RGB"))
    if a.ndim == 2:
        a = np.repeat(a[:, :, None], 3, axis=2)
    if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3:
        raise ValueError(f"expected uint8 [H,W,3] pixels, got {a.dtype} {a.shape}")
    return np.ascontiguousarray(a)


def pack_images(images):
    """-> (uint8 buffer, int64 offsets, int32 heights, int32 widths): the C-ABI batch layout of
    b200_preproc_run (images back to back, RGB uint8 HWC)."""
    arrs = [to_rgb8(im) for im in images]
    heights = np.array([a.shape[0] for a in arrs], np.int32)
    widths = np.array([a.shape[1] for a in arrs], np.int32)
    sizes = heights.astype(np.int64) * widths * 3
    offsets = np.zeros(len(arrs), np.int64)
    if len(arrs) > 1:
        offsets[1:] = np.cumsum(sizes[:-1])
    buf = np.empty(int(sizes.sum()), np.uint8)
    for a, o, s in zip(arrs, offsets, sizes):
        buf[o:o + s] = a.reshape(-1)
    return buf, offsets, heights, widths


class B200Preprocess:
    def __init__(self, n_px=224, mean=OPENAI_MEAN, std=OPENAI_STD, device=None, resize_mode="shortest"):
        if resize_mode not in RESIZE_MODES:
            raise ValueError("resize_mode %r: one of %s" % (resize_mode, ", ".join(RESIZE_MODES)))
        if device is None:
            device = torch.cuda.current_device() if torch.cuda.is_available() else 0
        self.device = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
        self.n_px = int(n_px)
        self.resize_mode = resize_mode
        m = (C.c_float * 3)(*mean)
        s = (C.c_float * 3)(*std)
        h = C.c_void_p()
        check(lib.b200_preproc_create_mode(self.n_px, m, s, RESIZE_MODES[resize_mode], self.device.index or 0,
                                           C.byref(h)))
        self._h = h

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            lib.b200_preproc_destroy(h)
        j, self._jpeg = getattr(self, "_jpeg", None), None
        if j:
            lib.b200_jpeg_destroy(j)

    def pack(self, images):
        return pack_images(images)

    def run_packed(self, pixels, offsets, heights, widths, out=None):
        """pixels: uint8 numpy buffer (host) or uint8 cuda tensor; returns float32 [n,3,n_px,n_px]."""
        n = len(heights)
        if out is None:
            out = torch.empty((n, 3, self.n_px, self.n_px), dtype=torch.float32, device=self.device)
        assert out.is_cuda and out.dtype == torch.float32 and out.is_contiguous() and out.shape[0] == n
        on_dev = isinstance(pixels, torch.Tensor) and pixels.is_cuda
        ptr = pixels.data_ptr() if isinstance(pixels, torch.Tensor) else pixels.ctypes.data
        offsets = np.ascontiguousarray(offsets, np.int64)
        heights = np.ascontiguousarray(heights, np.int32)
        widths = np.ascontiguousarray(widths, np.int32)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        check(lib.b200_preproc_run(self._h, C.c_void_p(ptr), int(on_dev), C.c_void_p(offsets.ctypes.data),
                                   C.c_void_p(heights.ctypes.data), C.c_void_p(widths.ctypes.data), n,
                                   C.c_void_p(out.data_ptr()), C.c_void_p(stream)))
        return out

    def __call__(self, images, out=None):
        if not isinstance(images, (list, tuple)):
            images = [images]
        return self.run_packed(*self.pack(images), out=out)

    # ---- JPEG bytes in (nvJPEG decode on the device) -----------------------------------------------------
    def from_jpeg_bytes(self, blobs, out=None):
        """blobs: list of bytes objects (JPEG files as read from disk / a tar shard, reader.py:98-106,158-165).
        Returns float32 [n, 3, n_px, n_px] on the device.  Images nvJPEG cannot parse (CMYK, progressive streams on
        some backends, non-JPEG files) are decoded with PIL on the host and uploaded as pixels."""
        import io

        n = len(blobs)
        if getattr(self, "_jpeg", None) is None:
            h = C.c_void_p()
            check(lib.b200_jpeg_create(self.device.index or 0, C.byref(h)), "jpeg_create")
            self._jpeg = h
        bufs = [np.frombuffer(b, dtype=np.uint8) for b in blobs]
        ptrs = (C.c_void_p * n)(*[b.ctypes.data for b in bufs])
        sizes = (C.c_size_t * n)(*[b.size for b in bufs])
        heights = np.zeros(n, np.int32)
        widths = np.zeros(n, np.int32)
        host = {}
        for i in range(n):   # per image, so that one unparsable stream does not fail the batch
            pi = (C.c_void_p * 1)(ptrs[i])
            si = (C.c_size_t * 1)(sizes[i])
            if lib.b200_jpeg_info(self._jpeg, pi, si, 1, C.c_void_p(heights[i:].ctypes.data), C.c_void_p(widths[i:].ctypes.data)) != 0:
                from PIL import Image

                host[i] = to_rgb8(Image.open(io.BytesIO(blobs[i])))
                heights[i], widths[i] = host[i].shape[0], host[i].shape[1]
        nbytes = heights.astype(np.int64) * widths * 3
        offsets = np.zeros(n, np.int64)
        if n > 1:
            offsets[1:] = np.cumsum(nbytes[:-1])
        pixels = torch.empty(int(nbytes.sum()), dtype=torch.uint8, device=self.device)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        dev_idx = [i for i in range(n) if i not in host]
        if dev_idx:
            k = len(dev_idx)
            p2 = (C.c_void_p * k)(*[ptrs[i] for i in dev_idx])
            s2 = (C.c_size_t * k)(*[sizes[i] for i in dev_idx])
            o2 = np.ascontiguousarray(offsets[dev_idx])
            h2 = np.ascontiguousarray(heights[dev_idx])
            w2 = np.ascontiguousarray(widths[dev_idx])
            check(lib.b200_jpeg_decode(self._jpeg, p2, s2, k, C.c_void_p(pixels.data_ptr()), C.c_void_p(o2.ctypes.data),
                                       C.c_void_p(h2.ctypes.data), C.c_void_p(w2.ctypes.data), C.c_void_p(stream)), "jpeg_decode")
        for i, a in host.items():
            pixels[offsets[i]:offsets[i] + nbytes[i]].copy_(torch.from_numpy(a.reshape(-1)))
        return self.run_packed(pixels, offsets, heights, widths, out=out)

    def decode_jpeg_bytes(self, blob):
        """One JPEG file -> uint8 [H, W, 3] numpy (device decode, copied back): for tests and inspection."""
        n = 1
        if getattr(self, "_jpeg", None) is None:
            h = C.c_void_p()
            check(lib.b200_jpeg_create(self.device.index or 0, C.byref(h)), "jpeg_create")
            self._jpeg = h
        buf = np.frombuffer(blob, dtype=np.uint8)
        ptrs = (C.c_void_p * n)(buf.ctypes.data)
        sizes = (C.c_size_t * n)(buf.size)
        hh, ww = np.zeros(1, np.int32), np.zeros(1, np.int32)
        check(lib.b200_jpeg_info(self._jpeg, ptrs, sizes, 1, C.c_void_p(hh.ctypes.data), C.c_void_p(ww.ctypes.data)), "jpeg_info")
        pixels = torch.empty(int(hh[0]) * int(ww[0]) * 3, dtype=torch.uint8, device=self.device)
        off = np.zeros(1, np.int64)
        check(lib.b200_jpeg_decode(self._jpeg, ptrs, sizes, 1, C.c_void_p(pixels.data_ptr()), C.c_void_p(off.ctypes.data),
                                   C.c_void_p(hh.ctypes.data), C.c_void_p(ww.ctypes.data),
                                   C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)), "jpeg_decode")
        return pixels.cpu().numpy().reshape(int(hh[0]), int(ww[0]), 3)
