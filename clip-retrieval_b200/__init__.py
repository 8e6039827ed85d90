"""b200clip — H100-native (sm_90a) hot path for rom1504/clip-retrieval.

Two paths, each behind the reference's own Python seam (SURVEY.md §8b):
  * search: `B200FlatIndex` / `B200IVFFlatIndex` / `B200IVFPQIndex` — the FAISS index object of
    clip_retrieval/clip_back.py:362 (`search`, `search_and_reconstruct`, `ntotal`, `d`, `nprobe`);
  * embed:  `load_clip` / `ClipMapper` — clip_retrieval/clip_inference/mapper.py:16-78, and the multilingual
    text towers behind `use_mclip` (`load_mclip`, `B200TextEncoder`; clip_back.py:836-859), and open_clip's
    XLM-RoBERTa CLIPs (`B200XLMRClip`, through `load_clip`), Google's SigLIP models (`SigLIPArch`) and
    open_clip's ConvNeXt CLIPs (`ConvNeXtArch`).
Everything numeric runs in the CUDA library `lib/libb200clip.so` (C ABI in include/b200clip.h);
there is no CPU fallback: importing works without a GPU, calling compute without one raises.
"""
from ._lib import lib, B200Error, library_path, launch_count  # noqa: F401
from .index import B200FlatIndex, B200IVFFlatIndex, B200IVFPQIndex, SynthSpec, load_index, merge_shard_results, merge_packed_results, train_kmeans, build_ivf_index, train_pq, train_ivfpq, build_ivfpq_index, train_opq  # noqa: F401
from .clip_index import clip_index, build_index, parse_index_key, default_index_key, default_nprobe  # noqa: F401
from .faiss_io import write_index, index_combiner  # noqa: F401

from .model import B200Clip, ClipArch, ResNetArch, SigLIPArch, ConvNeXtArch, Tower, ARCHS, G14_ARCHS, RESNET_ARCHS, SIGLIP_ARCHS, CONVNEXT_ARCHS, load_clip, synthetic_state_dict, convert_hf_state_dict  # noqa: F401,E402
from .preprocess import B200Preprocess, to_rgb8  # noqa: F401,E402
from .mclip import B200TextEncoder, EncoderArch, MCLIP_ARCHS, MclipTextModel, load_mclip  # noqa: F401,E402
from .xlmr_clip import B200XLMRClip, XLMRClipArch, XLMR_CLIP_ARCHS  # noqa: F401,E402
from .mapper import ClipMapper  # noqa: F401,E402
from .postfilter import get_non_uniques, get_violent_items, dedup_mask, H14NsfwDetector, get_unsafe_items  # noqa: F401,E402
from .service import B200KnnService, ClipResource, MicroBatcher  # noqa: F401,E402
from .sharded import ShardedIndex, B200ShardedIndex, shard_range  # noqa: F401,E402

__all__ = [
    "B200Clip", "ClipArch", "ResNetArch", "SigLIPArch", "ConvNeXtArch", "Tower", "ARCHS", "G14_ARCHS", "RESNET_ARCHS", "SIGLIP_ARCHS", "CONVNEXT_ARCHS", "load_clip", "synthetic_state_dict", "convert_hf_state_dict", "ClipMapper", "get_non_uniques", "get_violent_items", "dedup_mask", "H14NsfwDetector", "get_unsafe_items", "B200Preprocess", "to_rgb8", "B200KnnService", "ClipResource", "MicroBatcher", "ShardedIndex", "B200ShardedIndex", "shard_range",
    "lib", "B200Error", "library_path", "launch_count",
    "B200FlatIndex", "B200IVFFlatIndex", "B200IVFPQIndex", "SynthSpec", "load_index", "merge_shard_results", "train_kmeans", "build_ivf_index",
    "train_pq", "train_ivfpq", "build_ivfpq_index", "train_opq", "clip_index", "build_index", "parse_index_key",
    "default_index_key", "default_nprobe", "write_index", "index_combiner",
    "B200TextEncoder", "EncoderArch", "MCLIP_ARCHS", "MclipTextModel", "load_mclip",
    "B200XLMRClip", "XLMRClipArch", "XLMR_CLIP_ARCHS",
]
