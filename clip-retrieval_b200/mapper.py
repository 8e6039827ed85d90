"""Drop-in for the reference mapper (clip_retrieval/clip_inference/mapper.py:16-78).

Same constructor arguments, same `__call__(item) -> dict` contract (SURVEY.md §8b B1): `item`
carries `image_tensor` fp32 [B,3,S,S], `text_tokens` int [B,77], `image_filename`, `text`,
`metadata`; the result has the five keys `image_embs`, `text_embs`, `image_filename`, `text`,
`metadata`, with embeddings as np.float16 [B, D] arrays owned by Python (the writer keeps them
until flush: writer.py:43-56).  H2D copy, forward, L2-normalise, fp16 cast and D2H copy happen
inside one C-ABI call per modality (b200_clip_encode_image / b200_clip_encode_text).
With `use_mclip=True` the captions go through the multilingual encoder of `mclip_model` instead (mclip.py), and
`text_embs` are float32 normalized() rows as in the reference.

Extension (SURVEY §8(f) row 1): when the batch carries `image_rgb8` (a list of decoded uint8 HWC
images of any size — what a reader yields if its `preprocess` is `to_rgb8` instead of the torchvision
transform) instead of `image_tensor`, Resize/CenterCrop/ToTensor/Normalize run on the GPU
(`B200Preprocess`, bit-exact with the host transform, including its resize mode, mean and std:
`model.preprocess_params`) and feed the image tower in place.
"""
from .mclip import build_mclip
from .model import load_clip, preprocess_params
from .preprocess import B200Preprocess


class ClipMapper:
    """transforms images and texts into clip embeddings"""

    def __init__(
        self,
        enable_image,
        enable_text,
        enable_metadata,
        use_mclip,
        clip_model,
        use_jit,
        mclip_model,
        warmup_batch_size=1,
        clip_cache_path=None,
    ):
        self.enable_image = enable_image
        self.enable_text = enable_text
        self.enable_metadata = enable_metadata
        self.use_mclip = use_mclip
        self.mclip = None
        if use_mclip:
            # reference: SentenceTransformer(mclip_model).encode on the raw captions, then normalized()
            # (mapper.py:44-47,62-63): the text tower is replaced by the GPU encoder of that folder.  A name that is
            # no known encoder and no local folder raises NotImplementedError before anything is loaded.
            self.mclip = build_mclip(mclip_model, clip_cache_path, max_batch=max(int(warmup_batch_size), 32))
        self.device = "cuda"
        model, _, _ = load_clip(
            clip_model=clip_model,
            use_jit=use_jit,
            warmup_batch_size=warmup_batch_size,
            clip_cache_path=clip_cache_path,
        )
        self.model = model
        self._resize_mode, self._mean, self._std = preprocess_params(clip_model)
        self.model_img = model.encode_image
        self.model_txt = model.encode_text
        self._gpu_preprocess = None

    def __call__(self, item):
        image_embs = None
        text_embs = None
        image_filename = None
        text = None
        metadata = None
        if self.enable_image:
            if "image_tensor" not in item and "image_rgb8" in item:
                if self._gpu_preprocess is None:
                    self._gpu_preprocess = B200Preprocess(self.model.arch.image_size, mean=self._mean, std=self._std,
                                                          resize_mode=self._resize_mode)
                image_embs = self.model.embed_image(self._gpu_preprocess(item["image_rgb8"]))
            else:
                image_embs = self.model.embed_image(item["image_tensor"])
            image_filename = item["image_filename"]
        if self.enable_text:
            if self.use_mclip:
                text_embs = self.mclip.embed(item["text"])       # float32, as the reference's mclip path
            else:
                text_embs = self.model.embed_text(item["text_tokens"])
            text = item["text"]
        if self.enable_metadata:
            metadata = item["metadata"]
        return {
            "image_embs": image_embs,
            "text_embs": text_embs,
            "image_filename": image_filename,
            "text": text,
            "metadata": metadata,
        }
