"""open_clip's multilingual CLIPs with an XLM-RoBERTa text tower: `open_clip:xlm-roberta-base-ViT-B-32` and
`open_clip:xlm-roberta-large-ViT-H-14` (with or without a pretrained tag, or behind `synthetic:`).

What open_clip computes for them (DESIGN §5 (xv), recalled, not read from its source):
  * image: the CLIP ViT tower of `open_clip:ViT-B-32` / `open_clip:ViT-H-14` (erf GELU), `visual.*` keys;
  * text (`HFTextEncoder`, mean pooler, proj "mlp"): mask = ids != pad (1), h = XLMRobertaModel(ids, mask),
    pooled = (h * mask).sum(1) / mask.sum(1), out = Linear(d, h, no bias) -> GELU -> Linear(h, D, no bias) with
    h = (d + D) // 2; keys `text.transformer.*` (HuggingFace names), `text.proj.0.weight`, `text.proj.2.weight`;
  * tokenizer (`HFTokenizer`): whitespace_clean(basic_clean(text)), then the XLM-R tokenizer with max_length 77,
    padding to 77 with id 1, truncation (`</s>` stays last).
The image tower runs on an image-only `B200Clip` handle, the text tower on a `B200TextEncoder` with the MLP head.
For right-padded ids the key-length encoder (len[b] = first pad, positions 2 + t) is exactly the masked forward.
"""
import os
from dataclasses import dataclass, replace

import numpy as np

from . import mclip
from .model import ARCHS, B200Clip, Tower, _basic_clean, _find_checkpoint, _is_torch, _MissingTokenizer, \
    _whitespace_clean, make_preprocess, read_checkpoint, synthetic_state_dict as clip_synthetic_state_dict


@dataclass(frozen=True)
class XLMRClipArch:
    vision: object              # model.ClipArch of the image tower, text tower all zeros (an image-only handle)
    text: object                # mclip.EncoderArch, out_dim = embed_dim, no projection bias
    hidden: int                 # width of the MLP head: (text width + embed_dim) // 2
    tokenizer: str              # folder of tokenizer.json under clip_cache_path
    context_length: int = 77

    @property
    def embed_dim(self):
        return self.vision.embed_dim

    @property
    def image_size(self):
        return self.vision.image_size


_NO_TEXT = Tower(0, 0, 0, 0)
_XLMR = dict(family="xlm-roberta", vocab_size=250002, max_positions=514, type_vocab_size=1, pad_token_id=1,
             layer_norm_eps=1e-5, proj_bias=False)
XLMR_CLIP_ARCHS = {
    "xlm-roberta-base-ViT-B-32": XLMRClipArch(
        replace(ARCHS["open_clip:ViT-B-32"], text=_NO_TEXT),
        mclip.EncoderArch(layers=12, width=768, heads=12, ffn=3072, out_dim=512, **_XLMR), 640, "xlm-roberta-base"),
    "xlm-roberta-large-ViT-H-14": XLMRClipArch(
        replace(ARCHS["open_clip:ViT-H-14"], text=_NO_TEXT),
        mclip.EncoderArch(layers=24, width=1024, heads=16, ffn=4096, out_dim=1024, **_XLMR), 1024, "xlm-roberta-large"),
}


def resolve_xlmr_clip(clip_model):
    """(arch, key) when `clip_model` names one of XLMR_CLIP_ARCHS as `[synthetic:]open_clip:NAME[/PRETRAINED]`, else
    None (the name is for `model.resolve_arch`, which refuses unknown `open_clip:` names)."""
    name = clip_model[len("synthetic:"):] if clip_model.startswith("synthetic:") else clip_model
    if not name.startswith("open_clip:"):
        return None
    arch_name = name[len("open_clip:"):].partition("/")[0]
    if arch_name not in XLMR_CLIP_ARCHS:
        return None
    return XLMR_CLIP_ARCHS[arch_name], "open_clip:" + arch_name


# ---- weights ------------------------------------------------------------------------------------------------------

def _visual_shapes(v):
    w, t = v.vision.width, v.vision.mlp
    grid = v.image_size // v.patch
    out = {"visual.conv1.weight": (w, 3, v.patch, v.patch), "visual.class_embedding": (w,),
           "visual.positional_embedding": (grid * grid + 1, w), "visual.ln_pre.weight": (w,),
           "visual.ln_pre.bias": (w,), "visual.ln_post.weight": (w,), "visual.ln_post.bias": (w,),
           "visual.proj": (w, v.embed_dim)}
    for i in range(v.vision.layers):
        p = "visual.transformer.resblocks.%d." % i
        out.update({p + "ln_1.weight": (w,), p + "ln_1.bias": (w,), p + "attn.in_proj_weight": (3 * w, w),
                    p + "attn.in_proj_bias": (3 * w,), p + "attn.out_proj.weight": (w, w),
                    p + "attn.out_proj.bias": (w,), p + "ln_2.weight": (w,), p + "ln_2.bias": (w,),
                    p + "mlp.c_fc.weight": (t, w), p + "mlp.c_fc.bias": (t,), p + "mlp.c_proj.weight": (w, t),
                    p + "mlp.c_proj.bias": (w,)})
    return out


def _text_shapes(arch):
    """Key -> shape of the text encoder's layout (HuggingFace XLM-R names, projection.0 / projection.2)."""
    a = arch.text
    w, f = a.width, a.ffn
    out = {"embeddings.word_embeddings.weight": (a.vocab_size, w),
           "embeddings.position_embeddings.weight": (a.max_positions, w),
           "embeddings.token_type_embeddings.weight": (a.type_vocab_size, w),
           "embeddings.LayerNorm.weight": (w,), "embeddings.LayerNorm.bias": (w,),
           "projection.0.weight": (arch.hidden, w), "projection.2.weight": (a.out_dim, arch.hidden)}
    for i in range(a.layers):
        p = "encoder.layer.%d." % i
        for n in ("attention.self.query", "attention.self.key", "attention.self.value", "attention.output.dense"):
            out[p + n + ".weight"], out[p + n + ".bias"] = (w, w), (w,)
        out[p + "intermediate.dense.weight"], out[p + "intermediate.dense.bias"] = (f, w), (f,)
        out[p + "output.dense.weight"], out[p + "output.dense.bias"] = (w, f), (w,)
        for n in ("attention.output.LayerNorm", "output.LayerNorm"):
            out[p + n + ".weight"], out[p + n + ".bias"] = (w,), (w,)
    return out


def _text_key(k):
    """open_clip key -> the text encoder's key, or None for a key of no tower this model runs."""
    if k.startswith("text.transformer."):
        k = k[len("text.transformer."):]
        if k.startswith("pooler.") or k == "embeddings.position_ids":
            return None
        return k
    if k in ("text.proj.0.weight", "text.proj.2.weight"):
        return "projection" + k[len("text.proj"):]
    return None


def _checked(sd, shapes, where):
    for k, shape in shapes.items():
        if k not in sd:
            raise ValueError("%s: tensor %r is missing" % (where, k))
        if tuple(sd[k].shape) != tuple(shape):
            raise ValueError("%s: tensor %r has shape %s, expected %s" % (where, k, tuple(sd[k].shape), tuple(shape)))
    return {k: sd[k] for k in shapes}


def split_state_dict(sd, arch):
    """open_clip state_dict -> (image tower dict in B200Clip's `visual.*` layout, text dict in B200TextEncoder's
    layout).  The tensors are the same objects.  `logit_scale`, `text.transformer.pooler.*` and
    `text.transformer.embeddings.position_ids` are ignored; a missing or mis-shaped tensor raises ValueError naming
    its open_clip key."""
    visual = _checked({k: v for k, v in sd.items() if k.startswith("visual.")}, _visual_shapes(arch.vision),
                      "visual tower")
    text = {}
    for k, v in sd.items():
        t = _text_key(k)
        if t is not None:
            text[t] = v
    shapes = _text_shapes(arch)
    for k, shape in shapes.items():
        src = "text.proj" + k[len("projection"):] if k.startswith("projection.") else "text.transformer." + k
        if k not in text:
            raise ValueError("text tower: tensor %r is missing" % src)
        if tuple(text[k].shape) != tuple(shape):
            raise ValueError("text tower: tensor %r has shape %s, expected %s" % (src, tuple(text[k].shape), shape))
    return visual, {k: text[k] for k in shapes}


def synthetic_state_dict(arch, seed=0):
    """Seeded weights in open_clip's layout.  The `visual.*` tensors are those `model.synthetic_state_dict` gives the
    CLIP of the same image tower (it draws them first); the text tower is mclip's synthetic XLM-R plus the MLP head."""
    torch = mclip._torch()
    # any text tower gives the same visual draws; a one-width one keeps the discarded part small
    full = clip_synthetic_state_dict(replace(arch.vision, text=Tower(1, 0, 1, 1)), seed)
    sd = {k: v for k, v in full.items() if k.startswith("visual.")}
    text = mclip.synthetic_state_dict(replace(arch.text, out_dim=1), seed)
    del text["projection.weight"]
    g = torch.Generator().manual_seed(seed + 1)
    w, h, D = arch.text.width, arch.hidden, arch.embed_dim
    text["projection.0.weight"] = torch.randn(h, w, generator=g) * w ** -0.5
    text["projection.2.weight"] = torch.randn(D, h, generator=g) * h ** -0.5
    for k, v in text.items():
        sd["text.proj" + k[len("projection"):] if k.startswith("projection.") else "text.transformer." + k] = v
    sd["logit_scale"] = torch.tensor(4.6052)
    return sd


# ---- tokenizer ----------------------------------------------------------------------------------------------------

class XLMRTokenizer:
    """open_clip's HFTokenizer for these models: each text cleaned by whitespace_clean(basic_clean(.)), then the
    checkpoint's `tokenizer.json` with truncation to 77 tokens (special tokens included) and padding to 77 with the
    pad id.  texts -> LongTensor [n, 77].  `clean` and `context_length` replace the cleaning and the 77 (SigLIP's
    tokenizers: model.siglip_tokenizer)."""

    def __init__(self, path, pad_id=1, context_length=77, clean=None):
        try:
            from tokenizers import Tokenizer
        except ImportError as e:
            raise RuntimeError("the `tokenizers` package is needed to tokenize multilingual text") from e
        self.tok = Tokenizer.from_file(path)
        self.pad_id = int(pad_id)
        self.context_length = int(context_length)
        self.clean = clean or (lambda t: _whitespace_clean(_basic_clean(t)))
        self.tok.enable_truncation(max_length=self.context_length)
        self.tok.enable_padding(length=self.context_length, pad_id=self.pad_id,
                                pad_token=self.tok.id_to_token(self.pad_id) or "<pad>")

    def __call__(self, texts):
        torch = mclip._torch()
        if isinstance(texts, str):
            texts = [texts]
        encs = self.tok.encode_batch([self.clean(t) for t in texts])
        return torch.tensor([e.ids for e in encs], dtype=torch.long).reshape(len(encs), self.context_length)


def right_padded_lengths(ids, pad_id):
    """Token counts of right-padded rows ids [n, T] (host array).  ValueError naming the row when a non-pad id
    follows a pad id or when a row is all padding."""
    ids = np.asarray(ids)
    if ids.ndim != 2:
        raise ValueError("expected token ids [n, T], got shape %r" % (ids.shape,))
    pad = ids == pad_id
    lengths = np.where(pad.any(1), pad.argmax(1), ids.shape[1]).astype(np.int32)
    for r in range(ids.shape[0]):
        if lengths[r] == 0:
            raise ValueError("token row %d is all padding" % r)
        if not pad[r, lengths[r]:].all():
            raise ValueError("token row %d is not right-padded: a token follows the pad id %d at position %d"
                             % (r, pad_id, lengths[r]))
    return lengths


# ---- the model object ---------------------------------------------------------------------------------------------

class B200XLMRClip:
    """An open_clip XLM-RoBERTa CLIP on one GPU: an image-only `B200Clip` and a `B200TextEncoder` with the MLP
    head.  The surface of `B200Clip` that the mapper and the query service call: `encode_image` / `encode_text`
    (fp32 raw features), `embed_image[_device]` / `embed_text[_device]` (normalised rows, fp16 by default).  Text
    inputs are token ids [n, T] right-padded with the pad id (the tokenizer gives T = 77)."""

    def __init__(self, arch, device=0, max_batch=256):
        self.arch = arch
        self.device_index = int(device)
        self.visual = B200Clip(arch.vision, device=self.device_index, max_batch=max_batch)
        self.text = mclip.B200TextEncoder(arch.text, device=self.device_index, max_batch=max_batch,
                                          max_tokens=arch.context_length, mlp_hidden=arch.hidden)

    @property
    def device(self):
        return self.visual.device

    def load_state_dict(self, sd):
        """sd: open_clip state_dict (see split_state_dict)."""
        visual, text = split_state_dict(sd, self.arch)
        self.visual.load_state_dict(visual)
        self.text.load_state_dict(text)
        return self

    # ---- images: the image-only CLIP handle ----
    def encode_image(self, image):
        return self.visual.encode_image(image)

    def embed_image_device(self, image, dtype=None, normalize=True):
        return self.visual.embed_image_device(image, dtype, normalize)

    def embed_image(self, image_tensor):
        return self.visual.embed_image(image_tensor)

    # ---- text ----
    def encode_text(self, text):
        return self.embed_text_device(text, mclip._torch().float32, normalize=False)

    def embed_text_device(self, text, dtype=None, normalize=True):
        """ids [B, T] (right-padded) -> CUDA [B, D] (fp16 by default).  The token counts are computed on the device
        and the encoder runs the T it is given, so nothing waits for the host."""
        torch = mclip._torch()
        ids = torch.as_tensor(text).to(self.device, torch.int64).contiguous()
        if ids.dim() != 2:
            raise ValueError("embed_text: expected token ids [B, T], got %r" % (tuple(ids.shape),))
        lengths = torch.empty(ids.shape[0], dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            st = torch.cuda.current_stream(self.device).cuda_stream
            mclip.check(mclip.lib.b200_text_lengths_device(ids.data_ptr(), ids.shape[0], ids.shape[1],
                                                           self.arch.text.pad_token_id, lengths.data_ptr(), st),
                        "text_lengths")
        return self.text.embed_text_device(ids, lengths, dtype=dtype or torch.float16, normalize=normalize)

    def embed_text(self, text_tokens):
        """mapper.py:65-67 in one call: np.float16 [B, D], normalised.  Host ids are checked to be right-padded and
        the encoder runs on the batch's longest row only (bit-identical to running all 77 columns)."""
        if _is_torch(text_tokens):
            text_tokens = text_tokens.detach()
            if text_tokens.is_cuda:
                return self.embed_text_device(text_tokens).cpu().numpy()
            text_tokens = text_tokens.cpu().numpy()
        ids = np.ascontiguousarray(text_tokens, dtype=np.int64)
        lengths = right_padded_lengths(ids, self.arch.text.pad_token_id)
        T = int(lengths.max()) if len(lengths) else 1
        return self.text.embed_text(np.ascontiguousarray(ids[:, :T]), lengths, dtype=np.float16)


def read_xlmr_checkpoint(key, clip_cache_path, arch):
    """The open_clip state_dict of `<clip_cache_path>/<name>.{pt,pth,bin}` (model.py's rule for open_clip names)."""
    ckpt = _find_checkpoint(key, clip_cache_path)
    if ckpt is None:
        raise FileNotFoundError("no checkpoint for %r under clip_cache_path=%r (no network here); use 'synthetic:%s' "
                                "for seeded random weights" % (key, clip_cache_path, key))
    return read_checkpoint(ckpt, arch)


def load_xlmr_clip(clip_model, arch, key, warmup_batch_size, clip_cache_path, dev_index, max_batch):
    """load_clip's work for these names: (model, preprocess, tokenizer)."""
    torch = mclip._torch()
    if clip_model.startswith("synthetic:"):
        sd = synthetic_state_dict(arch, seed=0)
    else:
        sd = read_xlmr_checkpoint(key, clip_cache_path, arch)
    split_state_dict(sd, arch)                     # refuse a bad checkpoint before any device memory is taken
    model = B200XLMRClip(arch, device=dev_index, max_batch=max_batch).load_state_dict(sd)
    tp = os.path.join(clip_cache_path, arch.tokenizer, "tokenizer.json") if clip_cache_path else None
    if tp and os.path.exists(tp):
        tokenizer = XLMRTokenizer(tp, arch.text.pad_token_id, arch.context_length)
    else:
        tokenizer = _MissingTokenizer("no tokenizer.json for %r: expected <clip_cache_path>/%s/tokenizer.json"
                                      % (clip_model, arch.tokenizer))
    if warmup_batch_size and torch.cuda.is_available():
        wb = min(int(warmup_batch_size), max_batch)
        model.embed_image_device(torch.zeros(wb, 3, arch.image_size, arch.image_size, device=model.device))
        toks = torch.full((wb, arch.context_length), arch.text.pad_token_id, dtype=torch.long, device=model.device)
        toks[:, 0], toks[:, 1] = 0, 2
        model.embed_text_device(toks)
        torch.cuda.synchronize(model.device)
    return model, make_preprocess(arch.image_size), tokenizer
