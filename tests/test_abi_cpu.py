"""The C-ABI library loads without a GPU and exports every symbol include/b200clip.h declares;
the host-side mirrors fail loudly (no CPU fallback) when there is no device."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "b200clip.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    import clip_retrieval_b200 as m
    from clip_retrieval_b200 import _lib

    names = _declared()
    assert len(names) >= 35
    lib = ctypes.CDLL(m.library_path())
    for n in names:
        assert hasattr(lib, n), "library does not export %s" % n
        assert n in _lib.PROTOTYPES, "python binding has no prototype for %s" % n
    assert set(_lib.PROTOTYPES) == set(names)
    assert b"sm_90a" in _lib.lib.b200_version()


def test_no_cpu_fallback():
    import torch
    import clip_retrieval_b200 as m

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(m.B200Error):
        m.B200FlatIndex(768)
    with pytest.raises(m.B200Error):
        m.B200Clip(m.ARCHS["ViT-B/32"], max_batch=1)
    with pytest.raises(RuntimeError):
        m.load_clip("synthetic:ViT-B/32", device="cpu")


def test_arch_table_and_loader_errors():
    import clip_retrieval_b200 as m
    from clip_retrieval_b200.model import resolve_arch

    a, key = resolve_arch("open_clip:ViT-H-14/laion2b_s32b_b79k")
    assert key == "open_clip:ViT-H-14" and a.vision.width == 1280 and not a.quick_gelu
    assert resolve_arch("synthetic:ViT-L/14")[0].embed_dim == 768
    with pytest.raises(ValueError):
        resolve_arch("ViT-Z/99")
    sd = m.synthetic_state_dict(m.ClipArch(32, 32, 16, m.Tower(64, 1, 1, 128), m.Tower(64, 1, 1, 128)))
    assert sd["visual.conv1.weight"].shape == (64, 3, 16, 16) and sd["visual.positional_embedding"].shape == (5, 64)
    assert sd["transformer.resblocks.0.attn.in_proj_weight"].shape == (192, 64)


def test_shard_range_partitions_rows():
    import clip_retrieval_b200 as m

    for n, g in ((100, 8), (7, 8), (1_000_000_007, 8), (10, 3)):
        spans = [m.shard_range(n, g, r) for r in range(g)]
        assert spans[0][0] == 0 and spans[-1][1] == n
        assert all(spans[i][1] == spans[i + 1][0] for i in range(g - 1))
        sizes = [b - a for a, b in spans]
        assert max(sizes) - min(sizes) <= 1
