"""Generate tests/golden/clip_tiny-g14.npz with HuggingFace `transformers` CLIPModel, independent of oracle/clip_ref.py,
at a small config whose head dims are those of ViT-bigG-14's image tower (104) and ViT-g-14's (88), here on the text
tower so that the causal mask runs at head dim 88 too.  The weights are oracle.clip_ref.make_state_dict's (seed 0),
mapped to HF names by make_clip_golden.to_hf.  Run from the repo root:
    python tests/golden/make_g14_golden.py
The config is built here rather than in clip_ref.CONFIGS, whose `tiny*` keys feed other tests' parametrisations.
"""
import importlib.util
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import clip_ref  # noqa: E402

# vision 2 heads x 104 (T = 4^2 + 1 = 17), text 2 heads x 88 (T = 77), erf GELU as the LAION g / bigG checkpoints
CFG = clip_ref.ClipCfg(64, 56, 14, clip_ref.TowerCfg(208, 2, 2, 512), clip_ref.TowerCfg(176, 2, 2, 352),
                       quick_gelu=False, name="tiny-g14")
N = 5
OUT = os.path.join(ROOT, "tests", "golden", "clip_tiny-g14.npz")


def _make_clip_golden():
    spec = importlib.util.spec_from_file_location(
        "make_clip_golden", os.path.join(ROOT, "tests", "golden", "make_clip_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    torch.set_num_threads(8)
    gen = _make_clip_golden()
    sd = clip_ref.make_state_dict(CFG, seed=0)
    model = gen.to_hf(sd, CFG)
    px = clip_ref.synth_images(N, CFG, seed=0)
    tk = clip_ref.synth_tokens(N, CFG, seed=0)
    with torch.no_grad():
        fi = gen.feats(model.get_image_features(pixel_values=px)).float().numpy()
        ft = gen.feats(model.get_text_features(input_ids=tk, attention_mask=torch.ones_like(tk))).float().numpy()
    np.savez_compressed(OUT, image_features=fi, text_features=ft, n=N, seed=0, source="transformers CLIPModel fp32")
    oi = clip_ref.encode_image(sd, CFG, px).numpy()
    ot = clip_ref.encode_text(sd, CFG, tk).numpy()
    print("tiny-g14 HF vs oracle max abs diff: image %.3g text %.3g (|f| ~ %.3g)" % (
        np.abs(fi - oi).max(), np.abs(ft - ot).max(), np.abs(fi).mean()))


if __name__ == "__main__":
    main()
