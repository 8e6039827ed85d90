"""`open_clip:ViT-g-14` and `open_clip:ViT-bigG-14` without a GPU: how their names resolve, the table's figures, the
sharded HuggingFace snapshots their checkpoints come as, the HF key conversion at head dims 88 and 104, and the tower
oracle of tower_ref.py at their shapes, where it must accept an fp32 forward and reject the wrong forwards that only a
head dim of HD % 16 == 8 can have.  One of them, the softmax scale of the padded head dim, is 4 % off in the scores:
at two layers it stays inside the tower envelope (0.2-0.4 of the bound, measured), so it is shown rejected by the
per-element attention bound the kernel tests use instead.  Run with -s to see the ratios."""
import functools
import importlib.util
import json
import os
from dataclasses import replace

import pytest
import torch

import tower_ref as R
from oracle import clip_ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# name -> (embed dim, vision (width, layers, heads, mlp), text (width, layers, heads, mlp)): open_clip's ViT-g-14 and
# ViT-bigG-14 configs as recalled (DESIGN.md §5 (xvii)).  Both 224 px, patch 14, context 77, vocab 49408.
FIGURES = {
    "open_clip:ViT-g-14": (1024, (1408, 40, 16, 6144), (1024, 24, 16, 4096)),
    "open_clip:ViT-bigG-14": (1280, (1664, 48, 16, 8192), (1280, 32, 20, 5120)),
}


def _gen():
    spec = importlib.util.spec_from_file_location("make_clip_golden", os.path.join(GOLDEN, "make_clip_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


# ---- names ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name,arch_key,quick,key", [
    ("open_clip:ViT-g-14", "open_clip:ViT-g-14", False, "open_clip:ViT-g-14"),
    ("open_clip:ViT-g-14/laion2b_s12b_b42k", "open_clip:ViT-g-14", False, "open_clip:ViT-g-14"),
    ("open_clip:ViT-g-14/laion2b_s34b_b88k", "open_clip:ViT-g-14", False, "open_clip:ViT-g-14"),
    ("open_clip:ViT-g-14-quickgelu", "open_clip:ViT-g-14", True, "open_clip:ViT-g-14-quickgelu"),
    ("synthetic:open_clip:ViT-g-14/laion2b_s34b_b88k", "open_clip:ViT-g-14", False, "open_clip:ViT-g-14"),
    ("open_clip:ViT-bigG-14", "open_clip:ViT-bigG-14", False, "open_clip:ViT-bigG-14"),
    ("open_clip:ViT-bigG-14/laion2b_s39b_b160k", "open_clip:ViT-bigG-14", False, "open_clip:ViT-bigG-14"),
    ("open_clip:ViT-bigG-14-quickgelu", "open_clip:ViT-bigG-14", True, "open_clip:ViT-bigG-14-quickgelu"),
    ("synthetic:open_clip:ViT-bigG-14/laion2b_s39b_b160k", "open_clip:ViT-bigG-14", False, "open_clip:ViT-bigG-14"),
    ("hf_clip:laion/CLIP-ViT-g-14-laion2B-s12B-b42K", "open_clip:ViT-g-14", False,
     "hf_clip:laion/CLIP-ViT-g-14-laion2B-s12B-b42K"),
    ("hf_clip:laion/CLIP-ViT-g-14-laion2B-s34B-b88K", "open_clip:ViT-g-14", False,
     "hf_clip:laion/CLIP-ViT-g-14-laion2B-s34B-b88K"),
    ("hf_clip:laion/CLIP-ViT-bigG-14-laion2B-39B-b160k", "open_clip:ViT-bigG-14", False,
     "hf_clip:laion/CLIP-ViT-bigG-14-laion2B-39B-b160k"),
    ("synthetic:hf_clip:laion/CLIP-ViT-bigG-14-laion2B-39B-b160k", "open_clip:ViT-bigG-14", False,
     "hf_clip:laion/CLIP-ViT-bigG-14-laion2B-39B-b160k"),
])
def test_resolve_arch(name, arch_key, quick, key):
    import clip_retrieval_b200 as m
    from clip_retrieval_b200.model import _find_checkpoint, resolve_arch

    arch, got_key = resolve_arch(name)
    assert arch == replace(m.G14_ARCHS[arch_key], quick_gelu=quick)
    assert got_key == key
    assert _find_checkpoint(got_key, None) is None


@pytest.mark.parametrize("name,stem", [
    ("open_clip:ViT-g-14/laion2b_s34b_b88k", "ViT-g-14.pt"),
    ("open_clip:ViT-bigG-14/laion2b_s39b_b160k", "ViT-bigG-14.pth"),
    ("open_clip:ViT-bigG-14-quickgelu", "ViT-bigG-14-quickgelu.bin"),
])
def test_checkpoint_stem(tmp_path, name, stem):
    from clip_retrieval_b200.model import _find_checkpoint, resolve_arch

    _, key = resolve_arch(name)
    p = tmp_path / stem
    p.write_bytes(b"")
    assert _find_checkpoint(key, str(tmp_path)) == str(p)


def test_unknown_names_raise_and_list_both_tables():
    from clip_retrieval_b200.model import resolve_arch

    for bad in ("open_clip:ViT-G-14", "open_clip:ViT-bigg-14", "ViT-bigG-14", "hf_clip:laion/CLIP-ViT-bigG-14"):
        with pytest.raises(ValueError):
            resolve_arch(bad)
    with pytest.raises(ValueError) as e:
        resolve_arch("open_clip:nope")
    assert "open_clip:ViT-bigG-14" in str(e.value) and "open_clip:ViT-B-32" in str(e.value)


def test_existing_names_resolve_as_before():
    import clip_retrieval_b200 as m
    from clip_retrieval_b200.model import HF_REPOS, resolve_arch

    assert not set(m.ARCHS) & set(m.G14_ARCHS)
    for k, a in m.ARCHS.items():
        assert resolve_arch(k) == (a, k)
    for repo, (k, quick) in HF_REPOS.items():
        if k in m.ARCHS:
            assert resolve_arch("hf_clip:" + repo) == (replace(m.ARCHS[k], quick_gelu=quick), "hf_clip:" + repo)
    assert resolve_arch("open_clip:ViT-H-14/laion2b_s32b_b79k") == (m.ARCHS["open_clip:ViT-H-14"], "open_clip:ViT-H-14")


def test_table_matches_the_config_figures():
    import clip_retrieval_b200 as m

    assert set(m.G14_ARCHS) == set(FIGURES)
    for k, (D, v, t) in FIGURES.items():
        a = m.G14_ARCHS[k]
        assert a.embed_dim == D and (a.image_size, a.patch, a.context_length, a.vocab_size) == (224, 14, 77, 49408)
        assert not a.quick_gelu
        assert (a.vision.width, a.vision.layers, a.vision.heads, a.vision.mlp) == v
        assert (a.text.width, a.text.layers, a.text.heads, a.text.mlp) == t
        assert (a.image_size // a.patch) ** 2 + 1 == 257
    g, G = m.G14_ARCHS["open_clip:ViT-g-14"], m.G14_ARCHS["open_clip:ViT-bigG-14"]
    assert g.vision.width // g.vision.heads == 88 and G.vision.width // G.vision.heads == 104
    assert g.text.width // g.text.heads == 64 and G.text.width // G.text.heads == 64
    # open_clip's mlp_ratio -> int(width * ratio)
    assert int(1408 * 4.3637) == 6144 and int(1664 * 4.9231) == 8192


def test_hf_config_of_bigG_gives_the_table_entry():
    import clip_retrieval_b200 as m
    from clip_retrieval_b200.model import arch_from_hf_config

    def tower(t):
        return {"hidden_size": t.width, "num_hidden_layers": t.layers, "num_attention_heads": t.heads,
                "intermediate_size": t.mlp, "hidden_act": "gelu"}

    for a in m.G14_ARCHS.values():
        cfg = {"projection_dim": a.embed_dim,
               "vision_config": dict(tower(a.vision), image_size=224, patch_size=14),
               "text_config": dict(tower(a.text), max_position_embeddings=77, vocab_size=49408)}
        assert arch_from_hf_config(cfg) == a


# ---- checkpoints --------------------------------------------------------------------------------------------------------

# vision 2 heads x 104, text 2 heads x 88 (the golden's config, tests/golden/make_g14_golden.py) and the other way round
TINY = {
    "v104-t88": clip_ref.ClipCfg(64, 56, 14, clip_ref.TowerCfg(208, 2, 2, 512), clip_ref.TowerCfg(176, 2, 2, 352),
                                 quick_gelu=False, name="v104-t88"),
    "v88-t104": clip_ref.ClipCfg(64, 56, 14, clip_ref.TowerCfg(176, 2, 2, 352), clip_ref.TowerCfg(208, 2, 2, 512),
                                 quick_gelu=False, name="v88-t104"),
}


@pytest.mark.parametrize("name", list(TINY))
def test_convert_hf_state_dict_round_trips_at_head_dims_88_and_104(name):
    from clip_retrieval_b200.model import convert_hf_state_dict

    cfg = TINY[name]
    sd = clip_ref.make_state_dict(cfg, seed=0)
    back = convert_hf_state_dict(_gen().to_hf(sd, cfg).state_dict(), cfg)
    assert set(back) == set(sd) - {"logit_scale"}
    for k, v in back.items():
        assert v.shape == sd[k].shape and torch.equal(v, sd[k]), k


def _write_sharded(folder, hf_sd, kind, shards=3):
    """hf_sd split into `shards` files named as save_pretrained names them, plus the index."""
    keys = sorted(hf_sd)
    ext = "safetensors" if kind == "safetensors" else "bin"
    stem = "model" if kind == "safetensors" else "pytorch_model"
    weight_map = {}
    for i in range(shards):
        fname = "%s-%05d-of-%05d.%s" % (stem, i + 1, shards, ext)
        part = {k: hf_sd[k].contiguous().clone() for k in keys[i::shards]}
        if kind == "safetensors":
            from safetensors.torch import save_file

            save_file(part, os.path.join(folder, fname))
        else:
            torch.save(part, os.path.join(folder, fname))
        weight_map.update({k: fname for k in part})
    index = os.path.join(folder, "%s.%s.index.json" % (stem, ext))
    with open(index, "w") as f:
        json.dump({"metadata": {"total_size": 0}, "weight_map": weight_map}, f)
    return index


@pytest.mark.parametrize("kind", ["bin-sharded", "safetensors-sharded", "safetensors"])
def test_sharded_snapshot_reads_back_the_state_dict(tmp_path, kind):
    from clip_retrieval_b200.model import _find_checkpoint, read_checkpoint

    cfg = TINY["v104-t88"]
    sd = {k: v for k, v in clip_ref.make_state_dict(cfg, seed=0).items() if k != "logit_scale"}
    hf_sd = _gen().to_hf(clip_ref.make_state_dict(cfg, seed=0), cfg).state_dict()
    hf_sd = {k: v for k, v in hf_sd.items() if "position_ids" not in k}
    repo = "laion/CLIP-ViT-bigG-14-laion2B-39B-b160k"
    folder = tmp_path / repo
    folder.mkdir(parents=True)
    if kind == "safetensors":
        from safetensors.torch import save_file

        save_file({k: v.contiguous().clone() for k, v in hf_sd.items()}, str(folder / "model.safetensors"))
        want = str(folder / "model.safetensors")
    else:
        want = _write_sharded(str(folder), hf_sd, kind.split("-")[0])
    path = _find_checkpoint("hf_clip:" + repo, str(tmp_path))
    assert path == want
    got = read_checkpoint(path, cfg)
    assert set(got) == set(sd)
    for k, v in sd.items():
        assert got[k].dtype == v.dtype and torch.equal(got[k], v), (kind, k)
    if kind != "safetensors":
        # the sharded HF state_dict itself, before conversion, equals the unsharded one
        from clip_retrieval_b200.model import _read_sharded

        raw = _read_sharded(path)
        assert set(raw) == set(hf_sd) and all(torch.equal(raw[k], hf_sd[k]) for k in hf_sd)


def test_single_bin_is_still_preferred(tmp_path):
    from clip_retrieval_b200.model import _find_checkpoint

    repo = "laion/CLIP-ViT-g-14-laion2B-s12B-b42K"
    folder = tmp_path / repo
    folder.mkdir(parents=True)
    for f in ("pytorch_model.bin.index.json", "model.safetensors", "pytorch_model.bin"):
        (folder / f).write_bytes(b"")
    assert _find_checkpoint("hf_clip:" + repo, str(tmp_path)) == str(folder / "pytorch_model.bin")


# ---- tower oracle at the new shapes ---------------------------------------------------------------------------------------

def g14_cases():
    """name -> ClipArch at tower_ref.LAYERS blocks per tower: both G14_ARCHS entries and the quick-GELU bigG."""
    import clip_retrieval_b200 as m

    out = {}
    for k, a in m.G14_ARCHS.items():
        out[k] = a
    out["open_clip:ViT-bigG-14-quickgelu"] = replace(m.G14_ARCHS["open_clip:ViT-bigG-14"], quick_gelu=True)
    return {k: replace(a, vision=replace(a.vision, layers=R.LAYERS), text=replace(a.text, layers=R.LAYERS))
            for k, a in out.items()}


@functools.lru_cache(maxsize=2)
def g14_state_dict(name, weights="plain"):
    """clip_ref.make_state_dict of the case (seed 0), sensitised as tower_ref.state_dict does it."""
    sd = clip_ref.make_state_dict(R.clip_cfg(g14_cases()[name]), seed=0)
    return R.sensitise(sd) if weights == "sensitised" else sd


def _rows(t, head, dims, hd, plane):
    """Row indices of in_proj for dims `dims` of head `head` in plane 0 (q), 1 (k) or 2 (v)."""
    return [plane * t.width + head * hd + d for d in dims]


def mutate(sd, arch, mutation):
    """A copy of sd whose image tower computes one wrong forward of HD % 16 == 8 attention, through tower_ref.forward
    unchanged.  Every block's in_proj (weight and bias) is edited:
      qk_tail_dropped       q dims HD-8..HD-1 zero: the 8-wide QK^T tail left out
      out_tail_zeroed       v dims HD-8..HD-1 zero: the last n8 tile of P.V left out
      q_tail_from_next_head q dims HD-8..HD-1 of head h := dims 0..7 of the qkv columns after the head (head h+1's Q,
                            K of head 0 for the last head): a Q fragment loaded 8 columns too far"""
    t = arch.vision
    hd = t.width // t.heads
    tail = range(hd - 8, hd)
    out = dict(sd)
    for i in range(t.layers):
        for suffix in ("attn.in_proj_weight", "attn.in_proj_bias"):
            k = "visual.transformer.resblocks.%d.%s" % (i, suffix)
            x = sd[k].clone()
            for h in range(t.heads):
                if mutation == "qk_tail_dropped":
                    x[_rows(t, h, tail, hd, 0)] = 0.0
                elif mutation == "out_tail_zeroed":
                    x[_rows(t, h, tail, hd, 2)] = 0.0
                elif mutation == "q_tail_from_next_head":
                    x[_rows(t, h, tail, hd, 0)] = sd[k][[(h + 1) * hd + d for d in range(8)]]
                else:
                    raise ValueError(mutation)
            out[k] = x
    return out


# mutation -> (weight set, least worst-row ratio to the bound).  On the plain weights all three stay near the bound
# (measured 0.95-1.7): near-uniform attention averages the tail away.  On the sensitised weights (peaked attention) the
# worst rows over the three cases measured 5.35-6.90 (QK^T tail dropped), 2.81-3.91 (P.V tail zeroed) and 7.87-8.92
# (Q tail from the next head); the floors are at or below half of the smallest.
G14_REJECT_AT = {
    "qk_tail_dropped": ("sensitised", 2.5),
    "out_tail_zeroed": ("sensitised", 1.3),
    "q_tail_from_next_head": ("sensitised", 3.0),
}
SAMPLES = (0, 1)


@functools.lru_cache(maxsize=None)
def _results(name, weights):
    arch = g14_cases()[name]
    sd = g14_state_dict(name, weights)
    W = R.handle_weights(sd, "cpu")
    W32 = R.handle_weights(sd, "cpu", torch.float32)
    wrong = {m: R.handle_weights(mutate(sd, arch, m), "cpu", torch.float32)
             for m, (ws, _) in G14_REJECT_AT.items() if ws == weights}
    out = {"standin": [], "mutations": {m: [] for m in wrong}}
    for tower in ("image", "text"):
        for i in SAMPLES:
            x = R.sample(arch, tower, i)
            y, E = R.envelope(W, arch, tower, x)
            out["standin"].append(R.feature_ratio(R.forward(W32, arch, tower, x, dtype=torch.float32), y, E))
            if tower == "image":
                for m, Wm in wrong.items():
                    ym = R.forward(Wm, arch, tower, x, dtype=torch.float32)
                    out["mutations"][m].append(R.feature_ratio(ym, y, E))
    return out


def test_every_mutation_changes_the_image_in_proj_only():
    arch = g14_cases()["open_clip:ViT-g-14"]
    sd = g14_state_dict("open_clip:ViT-g-14")
    for m in G14_REJECT_AT:
        got = mutate(sd, arch, m)
        changed = {k for k in sd if not torch.equal(got[k], sd[k])}
        assert changed and all(k.startswith("visual.") and "in_proj" in k for k in changed), (m, changed)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("weights", R.WEIGHTS)
@pytest.mark.parametrize("name", list(g14_cases()))
def test_fp32_standin_is_inside_the_envelope(name, weights):
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    worst = max(_results(name, weights)["standin"])
    print("\n%-32s %-10s fp32 stand-in: worst |y - y_RN| / 2E = %.3f" % (name, weights, worst))
    assert worst <= 0.5, "a right forward with another summation order uses %.2f of the bound" % worst


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", list(g14_cases()))
@pytest.mark.parametrize("mutation", list(G14_REJECT_AT))
def test_wrong_forward_is_rejected(name, mutation):
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    weights, floor = G14_REJECT_AT[mutation]
    worst = max(_results(name, weights)["mutations"][mutation])
    print("\n%-32s %-22s %-10s worst ratio %7.2f (needs %4.1f)" % (name, mutation, weights, worst, floor))
    assert worst >= floor, "%s: the envelope accepts %s (ratio %.2f < %.1f)" % (name, mutation, worst, floor)


@pytest.mark.parametrize("hd", [88, 104])
def test_padded_scale_is_rejected_by_the_attention_bound(hd):
    """Softmax at (HD + 8)^-0.5, the scale of the padded head dim, against attention_ref64's per-element bound at the
    real image shape (T 257) on scores of the spread a trained tower has: far outside it."""
    from test_embed_gpu import attention_ref64

    T, heads = 257, 2
    w = heads * hd
    g = torch.Generator().manual_seed(hd)
    qkv = (torch.randn(T, 3 * w, generator=g) * torch.tensor([3.0, 3.0, 1.0]).repeat_interleave(w)).bfloat16()
    ref, bound, _ = attention_ref64(qkv, 1, T, heads, hd, 0)
    wrong = qkv.double().clone()
    wrong[:, :w] *= (hd / (hd + 8)) ** 0.5
    got, _, _ = attention_ref64(wrong, 1, T, heads, hd, 0)
    ratio = float(((got - ref).abs() / bound).max())
    print("\nhd %d: padded-scale softmax at %.1f x the attention bound" % (hd, ratio))
    assert ratio > 10.0
