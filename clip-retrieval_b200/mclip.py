"""Multilingual text towers on the GPU: what `use_mclip=True` selects in the mapper and the query service.

Reference seams:
  * query service: `load_mclip(clip_model)` (clip_back.py:836-859) -> a callable `text -> np.float32 [D]` built on
    M-CLIP `MultilingualCLIP` (XLM-RoBERTa-Large, masked mean pool, `LinearTransformation` with bias), followed by
    `normalized()` in `compute_query` (clip_back.py:222-224);
  * mapper: `SentenceTransformer(mclip_model).encode(texts)` (mapper.py:44-47,62-63; DistilBERT, mean pooling, Dense
    without activation), followed by `normalized()`; the embeddings stay float32.
The encoder runs in the CUDA library (include/b200clip.h, b200_text_encoder_*).  Tokenisation is host plumbing: the
checkpoint's own `tokenizer.json` through the `tokenizers` package (what `transformers.AutoTokenizer` runs), with
padding and truncation set as the reference call sites set them.
Weights come from local folders (no downloads): `<clip_cache_path>/<repo>/` (a HuggingFace snapshot folder) or
`<clip_cache_path>/<repo with / replaced by ->/`, or a folder path; `synthetic:<repo>` gives seeded random weights.
"""
import ctypes as C
import json
import os
import threading
from dataclasses import dataclass, replace
from functools import lru_cache

import numpy as np

from . import _lib
from ._lib import lib, check


@dataclass(frozen=True)
class EncoderArch:
    family: str                 # "xlm-roberta" | "distilbert"
    layers: int
    width: int
    heads: int
    ffn: int
    vocab_size: int
    max_positions: int
    type_vocab_size: int        # 0: no token-type table
    pad_token_id: int
    layer_norm_eps: float
    out_dim: int
    proj_bias: bool
    max_seq_length: int = 0     # > 0: truncate to this many tokens (SentenceTransformer); 0: no truncation (M-CLIP)

    @property
    def position_offset(self):
        # XLM-R numbers the tokens of a sample from padding_idx + 1; DistilBERT from 0
        return self.pad_token_id + 1 if self.family == "xlm-roberta" else 0

    @property
    def max_tokens(self):
        return min(self.max_positions - self.position_offset, 512)


_XLMR_LARGE = dict(family="xlm-roberta", layers=24, width=1024, heads=16, ffn=4096, vocab_size=250002,
                   max_positions=514, type_vocab_size=1, pad_token_id=1, layer_norm_eps=1e-5, proj_bias=True)
MCLIP_ARCHS = {
    "M-CLIP/XLM-Roberta-Large-Vit-L-14": EncoderArch(out_dim=768, **_XLMR_LARGE),
    "M-CLIP/XLM-Roberta-Large-Vit-B-32": EncoderArch(out_dim=512, **_XLMR_LARGE),
    "sentence-transformers/clip-ViT-B-32-multilingual-v1": EncoderArch(
        "distilbert", 6, 768, 12, 3072, 119547, 512, 0, 0, 1e-12, 512, False, max_seq_length=128),
}
# clip_back.load_mclip's choice of the M-CLIP model for the CLIP model a back end serves
CLIP_TO_MCLIP = {"ViT-L/14": "M-CLIP/XLM-Roberta-Large-Vit-L-14", "ViT-B/32": "M-CLIP/XLM-Roberta-Large-Vit-B-32"}
ACCEPTED = ("a repository of the table (%s) with its folder under clip_cache_path as <repo>/ or <repo with / -> ->/; "
            "synthetic:<repo>; or the path of an M-CLIP folder (config.json with modelBase, transformerDimensions, "
            "numDims) or a SentenceTransformer folder (DistilBERT module, mean pooling, Dense without activation)"
            % ", ".join(sorted(MCLIP_ARCHS)))


def _torch():
    import torch

    return torch


# ---- weights ------------------------------------------------------------------------------------------------------

def synthetic_state_dict(arch, seed=0):
    """Seeded random weights (normal, std 0.02: BERT's init scale) in the key layout `load_state_dict` takes."""
    torch = _torch()
    g = torch.Generator().manual_seed(seed)

    def rn(*shape, std=0.02):
        return torch.randn(*shape, generator=g, dtype=torch.float32) * std

    w = arch.width
    sd = {"embeddings.word_embeddings.weight": rn(arch.vocab_size, w),
          "embeddings.position_embeddings.weight": rn(arch.max_positions, w),
          "embeddings.LayerNorm.weight": 1.0 + rn(w, std=0.1), "embeddings.LayerNorm.bias": rn(w, std=0.05)}
    if arch.type_vocab_size:
        sd["embeddings.token_type_embeddings.weight"] = rn(arch.type_vocab_size, w)
    for i in range(arch.layers):
        p = "encoder.layer.%d." % i
        for n in ("attention.self.query", "attention.self.key", "attention.self.value", "attention.output.dense"):
            sd[p + n + ".weight"], sd[p + n + ".bias"] = rn(w, w), rn(w)
        sd[p + "intermediate.dense.weight"], sd[p + "intermediate.dense.bias"] = rn(arch.ffn, w), rn(arch.ffn)
        sd[p + "output.dense.weight"], sd[p + "output.dense.bias"] = rn(w, arch.ffn), rn(w)
        for n in ("attention.output.LayerNorm", "output.LayerNorm"):
            sd[p + n + ".weight"], sd[p + n + ".bias"] = 1.0 + rn(w, std=0.1), rn(w, std=0.05)
    sd["projection.weight"] = rn(arch.out_dim, w, std=w ** -0.5)
    if arch.proj_bias:
        sd["projection.bias"] = rn(arch.out_dim)
    return sd


_DISTILBERT_NAMES = (("attention.q_lin", "attention.self.query"), ("attention.k_lin", "attention.self.key"),
                     ("attention.v_lin", "attention.self.value"), ("attention.out_lin", "attention.output.dense"),
                     ("sa_layer_norm", "attention.output.LayerNorm"), ("ffn.lin1", "intermediate.dense"),
                     ("ffn.lin2", "output.dense"), ("output_layer_norm", "output.LayerNorm"))


def convert_distilbert_state_dict(sd):
    """HuggingFace DistilBertModel names -> the BERT layout (`transformer.layer.N.attention.q_lin` ->
    `encoder.layer.N.attention.self.query`, ...)."""
    out = {}
    for k, v in sd.items():
        if k.startswith("transformer.layer."):
            i, rest = k[len("transformer.layer."):].split(".", 1)
            for a, b in _DISTILBERT_NAMES:
                if rest.startswith(a + "."):
                    rest = b + rest[len(a):]
                    break
            k = "encoder.layer.%s.%s" % (i, rest)
        out[k] = v
    return out


def _read_weights(folder):
    """state_dict of `model.safetensors` or `pytorch_model.bin` in `folder`."""
    p = os.path.join(folder, "model.safetensors")
    if os.path.exists(p):
        from safetensors.torch import load_file

        return load_file(p)
    p = os.path.join(folder, "pytorch_model.bin")
    if os.path.exists(p):
        return _torch().load(p, map_location="cpu", weights_only=True)
    raise FileNotFoundError("no model.safetensors or pytorch_model.bin in %s" % folder)


def _json(path):
    with open(path) as f:
        return json.load(f)


def _hf_arch(cfg, out_dim, proj_bias, max_seq_length=0):
    """EncoderArch of a HuggingFace XLM-R / DistilBERT config.json dict (eps from the config, never a default)."""
    mt = cfg.get("model_type")
    if mt == "xlm-roberta":
        return EncoderArch("xlm-roberta", int(cfg["num_hidden_layers"]), int(cfg["hidden_size"]),
                           int(cfg["num_attention_heads"]), int(cfg["intermediate_size"]), int(cfg["vocab_size"]),
                           int(cfg["max_position_embeddings"]), int(cfg.get("type_vocab_size", 1)),
                           int(cfg.get("pad_token_id", 1)), float(cfg["layer_norm_eps"]), out_dim, proj_bias,
                           max_seq_length)
    if mt == "distilbert":
        if cfg.get("sinusoidal_pos_embds"):
            raise NotImplementedError("DistilBERT with sinusoidal position embeddings is not supported")
        # DistilBERT's LayerNorms are built with eps 1e-12 whatever the config says
        return EncoderArch("distilbert", int(cfg["n_layers"]), int(cfg["dim"]), int(cfg["n_heads"]),
                           int(cfg["hidden_dim"]), int(cfg["vocab_size"]), int(cfg["max_position_embeddings"]), 0,
                           int(cfg.get("pad_token_id", 0)), 1e-12, out_dim, proj_bias, max_seq_length)
    raise NotImplementedError("text encoder model_type %r is not supported (xlm-roberta, distilbert)" % mt)


def read_mclip_folder(folder):
    """M-CLIP folder: config.json (MCLIPConfig: modelBase, transformerDimensions, numDims), weights with keys
    `transformer.*` (XLMRobertaModel) and `LinearTransformation.{weight,bias}`.  -> (arch, state_dict)."""
    cfg = _json(os.path.join(folder, "config.json"))
    base = cfg.get("modelBase", "")
    if "xlm-roberta" not in base:
        raise NotImplementedError("M-CLIP modelBase %r is not supported (xlm-roberta-large)" % base)
    raw = _read_weights(folder)
    sd = {k[len("transformer."):]: v for k, v in raw.items() if k.startswith("transformer.")}
    sd["projection.weight"] = raw["LinearTransformation.weight"]
    if "LinearTransformation.bias" in raw:
        sd["projection.bias"] = raw["LinearTransformation.bias"]
    # the XLM-R config itself is not in the folder (MultilingualCLIP builds it from modelBase): shapes come from the
    # weights, eps and the pad id from xlm-roberta-large's config
    word, pos = sd["embeddings.word_embeddings.weight"], sd["embeddings.position_embeddings.weight"]
    layers = len({k.split(".")[2] for k in sd if k.startswith("encoder.layer.")})
    width = int(word.shape[1])
    if width != int(cfg.get("transformerDimensions", width)) or int(cfg["numDims"]) != sd["projection.weight"].shape[0]:
        raise ValueError("M-CLIP folder %s: config.json does not match the weights" % folder)
    tt = sd.get("embeddings.token_type_embeddings.weight")
    arch = replace(MCLIP_ARCHS["M-CLIP/XLM-Roberta-Large-Vit-L-14"], layers=layers, width=width, heads=width // 64,
                   ffn=int(sd["encoder.layer.0.intermediate.dense.weight"].shape[0]), vocab_size=int(word.shape[0]),
                   max_positions=int(pos.shape[0]), type_vocab_size=0 if tt is None else int(tt.shape[0]),
                   out_dim=int(cfg["numDims"]), proj_bias="projection.bias" in sd)
    return arch, sd


def read_st_folder(folder):
    """SentenceTransformer folder: modules.json listing a Transformer (DistilBERT), a Pooling (mean only) and a Dense
    (Identity activation) module; sentence_bert_config.json gives max_seq_length.  -> (arch, state_dict)."""
    mods = _json(os.path.join(folder, "modules.json"))
    by_type = {m["type"].rsplit(".", 1)[-1]: os.path.join(folder, m.get("path", "")) for m in mods}
    if set(by_type) != {"Transformer", "Pooling", "Dense"}:
        raise NotImplementedError("SentenceTransformer modules %s: only Transformer + Pooling + Dense is supported"
                                  % sorted(by_type))
    pool = _json(os.path.join(by_type["Pooling"], "config.json"))
    modes = sorted(k for k, v in pool.items() if k.startswith("pooling_mode") and v)
    if modes != ["pooling_mode_mean_tokens"]:
        raise NotImplementedError("SentenceTransformer pooling %s: only mean pooling is supported" % modes)
    dense = _json(os.path.join(by_type["Dense"], "config.json"))
    act = dense.get("activation_function", "torch.nn.modules.linear.Identity")
    if not act.endswith("Identity"):
        raise NotImplementedError("SentenceTransformer Dense activation %r: only Identity is supported" % act)
    tdir = by_type["Transformer"]
    st_cfg_path = os.path.join(tdir, "sentence_bert_config.json")
    if not os.path.exists(st_cfg_path):
        st_cfg_path = os.path.join(folder, "sentence_bert_config.json")
    max_seq = int(_json(st_cfg_path).get("max_seq_length", 0) or 0)
    sd = _read_weights(tdir)
    if any(k.startswith("transformer.layer.") for k in sd):
        sd = convert_distilbert_state_dict(sd)
    dsd = _read_weights(by_type["Dense"])
    sd["projection.weight"] = dsd["linear.weight"]
    bias = bool(dense.get("bias", "linear.bias" in dsd))
    if bias:
        sd["projection.bias"] = dsd["linear.bias"]
    arch = _hf_arch(_json(os.path.join(tdir, "config.json")), int(dense["out_features"]), bias, max_seq)
    return arch, sd


def _tokenizer_path(folder):
    for sub in ("", "0_Transformer"):
        p = os.path.join(folder, sub, "tokenizer.json")
        if os.path.exists(p):
            return p
    return None


def resolve_mclip(name, clip_cache_path=None):
    """(arch, state_dict or None for synthetic weights, folder or None) for an mclip model name.  Raises
    NotImplementedError for a name that is neither a known repository, `synthetic:<repo>` nor a model folder."""
    if name.startswith("synthetic:"):
        repo = name[len("synthetic:"):]
        if repo not in MCLIP_ARCHS:
            raise NotImplementedError("mclip model %r is not supported; accepted: %s" % (name, ACCEPTED))
        return MCLIP_ARCHS[repo], None, None
    folder = None
    if os.path.isdir(name):
        folder = name
    elif name in MCLIP_ARCHS:
        for cand in (name, name.replace("/", "-")):
            p = os.path.join(clip_cache_path, cand) if clip_cache_path else None
            if p and os.path.isdir(p):
                folder = p
                break
        if folder is None:
            raise FileNotFoundError("no folder for %r under clip_cache_path=%r (no network here); use 'synthetic:%s' "
                                    "for seeded random weights" % (name, clip_cache_path, name))
    else:
        raise NotImplementedError("mclip model %r is not supported; accepted: %s" % (name, ACCEPTED))
    if os.path.exists(os.path.join(folder, "modules.json")):
        arch, sd = read_st_folder(folder)
    else:
        arch, sd = read_mclip_folder(folder)
    return arch, sd, folder


# ---- tokenizer ----------------------------------------------------------------------------------------------------

class MclipTokenizer:
    """The checkpoint's `tokenizer.json` through `tokenizers`, called as the reference calls it: padding to the
    longest text of the call, truncation to `max_length` when given (SentenceTransformer), none otherwise (M-CLIP).
    texts -> (ids int64 [n, T], lengths int32 [n]), right-padded with the pad id."""

    def __init__(self, path, arch):
        try:
            from tokenizers import Tokenizer
        except ImportError as e:
            raise RuntimeError("the `tokenizers` package is needed to tokenize multilingual text") from e
        self.tok = Tokenizer.from_file(path)
        self.pad_id = arch.pad_token_id
        self.max_tokens = arch.max_tokens
        self.tok.no_padding()
        if arch.max_seq_length:
            self.tok.enable_truncation(max_length=arch.max_seq_length, strategy="longest_first")
        else:
            self.tok.no_truncation()

    def __call__(self, texts):
        if isinstance(texts, str):
            texts = [texts]
        encs = self.tok.encode_batch(list(texts))
        lengths = np.array([len(e.ids) for e in encs], dtype=np.int32)
        if lengths.max() > self.max_tokens:
            raise ValueError("text of %d tokens is longer than the %d positions the model has"
                             % (int(lengths.max()), self.max_tokens))
        ids = np.full((len(encs), int(lengths.max())), self.pad_id, dtype=np.int64)
        for i, e in enumerate(encs):
            ids[i, :len(e.ids)] = e.ids
        return ids, lengths


class _MissingTokenizer:
    def __init__(self, why):
        self.why = why

    def __call__(self, texts):
        raise RuntimeError(self.why)


# ---- the encoder --------------------------------------------------------------------------------------------------

class B200TextEncoder:
    """A BERT-family text encoder on one GPU (b200_text_encoder_*).  Inputs are right-padded ids [B, T] and the
    per-sample token counts; padding never changes a sample's result.  `mlp_hidden` > 0 selects open_clip's MLP head
    (width -> mlp_hidden -> out_dim, GELU between, no biases; weights projection.0.weight / projection.2.weight)
    instead of the linear projection."""

    def __init__(self, arch, device=0, max_batch=64, max_tokens=None, mlp_hidden=0):
        self.arch = arch
        self.mlp_hidden = int(mlp_hidden)
        self.device_index = int(device)
        self.max_batch = int(max_batch)
        self.max_tokens = int(max_tokens or arch.max_tokens)
        self._h = C.c_void_p()
        self._lock = threading.Lock()
        cfg = _lib.TextEncoderConfigC(arch.layers, arch.width, arch.heads, arch.ffn, arch.vocab_size,
                                      arch.max_positions, arch.type_vocab_size, arch.position_offset,
                                      arch.layer_norm_eps, arch.out_dim, 1 if arch.proj_bias else 0,
                                      self.max_batch, self.max_tokens)
        if self.mlp_hidden:
            check(lib.b200_text_encoder_create_mlp(C.byref(cfg), self.mlp_hidden, self.device_index, C.byref(self._h)),
                  "text_encoder_create_mlp")
        else:
            check(lib.b200_text_encoder_create(C.byref(cfg), self.device_index, C.byref(self._h)), "text_encoder_create")

    def __del__(self):
        try:
            if self._h:
                lib.b200_text_encoder_destroy(self._h)
                self._h = C.c_void_p()
        except Exception:
            pass

    @property
    def device(self):
        return _torch().device("cuda", self.device_index)

    def load_state_dict(self, sd):
        """sd: name -> tensor / array (fp32 or fp16) in the BERT key layout plus projection.{weight,bias}."""
        from .model import _tensor_views

        views, keep = _tensor_views(sd)
        check(lib.b200_text_encoder_load_weights(self._h, views, len(keep)), "text_encoder_load_weights")
        return self

    def embed_text_device(self, ids, lengths, dtype=None, normalize=True):
        """ids int [B, T], lengths int [B] (1..T) -> CUDA [B, out_dim] (fp32 by default), normalized() rows unless
        `normalize` is False.  Asynchronous on the current stream."""
        torch = _torch()
        ids = torch.as_tensor(ids).to(self.device, torch.int64).contiguous()
        lengths = torch.as_tensor(lengths).to(self.device, torch.int32).contiguous()
        if ids.dim() != 2 or lengths.shape != (ids.shape[0],):
            raise ValueError("embed_text_device: ids [B, T] and lengths [B], got %r and %r"
                             % (tuple(ids.shape), tuple(lengths.shape)))
        dtype = dtype or torch.float32
        B, T = ids.shape
        out = torch.empty((B, self.arch.out_dim), dtype=dtype, device=self.device)
        st = torch.cuda.current_stream(self.device).cuda_stream
        with self._lock:
            check(lib.b200_text_encoder_encode_device(self._h, ids.data_ptr(), lengths.data_ptr(), B, T, out.data_ptr(),
                                                      1 if dtype == torch.float16 else 0, 1 if normalize else 0, st),
                  "text_encoder_encode")
        return out

    def embed_text(self, ids, lengths, normalize=True, dtype=np.float32):
        """Host arrays in, np.float32 (or `dtype` np.float16) [B, out_dim] out (H2D, forward, D2H in one library
        call)."""
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        lengths = np.ascontiguousarray(lengths, dtype=np.int32)
        if ids.ndim != 2 or lengths.shape != (ids.shape[0],):
            raise ValueError("embed_text: ids [B, T] and lengths [B], got %r and %r" % (ids.shape, lengths.shape))
        out = np.empty((ids.shape[0], self.arch.out_dim), dtype=dtype)
        check(lib.b200_text_encoder_encode(self._h, ids.ctypes.data, lengths.ctypes.data, ids.shape[0], ids.shape[1],
                                           out.ctypes.data, 1 if out.dtype == np.float16 else 0, 1 if normalize else 0),
              "text_encoder_encode")
        return out

    def set_profiling(self, on):
        check(lib.b200_text_encoder_set_profiling(self._h, 1 if on else 0), "set_profiling")

    def last_timing(self):
        ms = (C.c_float * 4)()
        n = C.c_int(0)
        check(lib.b200_text_encoder_last_timing(self._h, ms, C.byref(n)), "last_timing")
        return {"gemm": ms[0], "attention": ms[1], "layernorm": ms[2], "other": ms[3], "launches": int(n.value)}


class MclipTextModel:
    """Encoder + tokenizer.  Called with one text it is clip_back.load_mclip's `encode_texts`: raw fp32 features
    [out_dim] on the host.  `embed_device` keeps normalized() rows on the device for the search that follows."""

    def __init__(self, encoder, tokenizer):
        self.encoder = encoder
        self.tokenizer = tokenizer

    def __call__(self, text):
        ids, lengths = self.tokenizer([text])
        return self.encoder.embed_text(ids, lengths, normalize=False)[0]

    def embed_device(self, texts=None, tokens=None):
        """normalized() fp32 CUDA rows [n, out_dim] of `texts`, or of pre-tokenised `tokens` = (ids, lengths)."""
        ids, lengths = tokens if tokens is not None else self.tokenizer(texts)
        return self.encoder.embed_text_device(ids, lengths)

    def embed(self, texts):
        """normalized() np.float32 rows [n, out_dim] (the mapper's `text_embs`)."""
        ids, lengths = self.tokenizer(texts)
        return self.encoder.embed_text(ids, lengths)


def build_mclip(name, clip_cache_path=None, device=None, max_batch=64):
    """MclipTextModel for an mclip model name (see ACCEPTED)."""
    torch = _torch()
    arch, sd, folder = resolve_mclip(name, clip_cache_path)
    if device is None:
        dev_index = torch.cuda.current_device() if torch.cuda.is_available() else 0
    else:
        d = torch.device(device)
        if d.type != "cuda":
            raise RuntimeError("b200clip has no CPU path: device=%r" % (device,))
        dev_index = d.index if d.index is not None else torch.cuda.current_device()
    enc = B200TextEncoder(arch, device=dev_index, max_batch=max_batch)
    enc.load_state_dict(sd if sd is not None else synthetic_state_dict(arch, seed=0))
    tp = _tokenizer_path(folder) if folder else None
    tok = MclipTokenizer(tp, arch) if tp else _MissingTokenizer("no tokenizer.json for mclip model %r" % name)
    return MclipTextModel(enc, tok)


@lru_cache(maxsize=None)
def load_mclip(clip_model, clip_cache_path=None, device=None):
    """Drop-in for clip_back.load_mclip: the M-CLIP text model for the CLIP model a back end serves ("ViT-L/14" ->
    M-CLIP/XLM-Roberta-Large-Vit-L-14, "ViT-B/32" -> ...-Vit-B-32; a `synthetic:` prefix selects seeded weights).
    An mclip model name or folder (see ACCEPTED) is taken as is.  Returns a callable text -> np.float32 [D]."""
    synthetic = clip_model.startswith("synthetic:")
    base = clip_model[len("synthetic:"):] if synthetic else clip_model
    if base in CLIP_TO_MCLIP:
        name = ("synthetic:" if synthetic else "") + CLIP_TO_MCLIP[base]
    elif base in MCLIP_ARCHS or os.path.isdir(base):
        name = clip_model
    else:
        raise ValueError("Multi-lingual version of %s not available." % clip_model)
    return build_mclip(name, clip_cache_path, device, max_batch=8)
