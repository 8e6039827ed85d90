"""Writes tests/golden/reference_calls.json: what the original clip-retrieval code returns on the seeded inputs of
tests/test_oracle_cpu.py and tests/test_preprocess_cpu.py, so that those tests compare the oracle with it without the
original checkout.  Run once where the checkout exists:  python tests/golden/make_reference_golden.py /path/to/clip-retrieval
  * KnnService.connected_components / get_violent_items / knn_search (+ post_filter, normalized), clip_back.py,
    extracted with ast and executed unmodified;
  * ClipMapper.__call__ (mapper.py) on fixed seeded features;
  * sha256 of every tensor of tests/test_clip_inference/test_tensors/*.pkl (their JPEGs are in golden/ref_images)."""
import ast
import contextlib
import glob
import hashlib
import json
import os
import pickle
import sys
import textwrap
import types
from collections import defaultdict

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import knn_ref, synth_ref  # noqa: E402
from oracle import postfilter_ref as R  # noqa: E402


def postfilter_inputs():
    """The seeded graphs / prompt sets of test_postfilter_oracle_matches_reference_functions."""
    rng = np.random.default_rng(0)
    graphs = []
    for _ in range(20):
        k = int(rng.integers(2, 60))
        A = rng.random((k, k)) < 0.05
        graphs.append(A | A.T | np.eye(k, dtype=bool))
    E = rng.standard_normal((200, 64)).astype(np.float32)
    P = rng.standard_normal((3, 64)).astype(np.float32)
    return graphs, E, P


def neighbours(A):
    neigh = defaultdict(list)
    for i in range(A.shape[0]):
        for j in np.nonzero(A[i])[0]:
            neigh[int(i)].append(int(j))
    return neigh


def mapper_features():
    g = torch.Generator().manual_seed(11)
    return torch.randn(5, 32, generator=g), torch.randn(5, 32, generator=g)


def index_contract_rows():
    X = synth_ref.rows_f16(30, 64)
    X[7] = X[3]
    return X


def main(ref):
    out = {}
    src = open(os.path.join(ref, "clip_retrieval", "clip_back.py")).read()
    tree = ast.parse(src)
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "KnnService")
    timer = types.SimpleNamespace(time=lambda: contextlib.nullcontext())
    ns = {"np": np, "KNN_INDEX_TIME": timer, "DEDUP_TIME": timer, "SAFETY_TIME": timer}
    exec(ast.get_source_segment(src, next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "normalized")), ns)
    for node in cls.body:
        if isinstance(node, ast.FunctionDef) and node.name in ("connected_components", "get_violent_items", "knn_search",
                                                                "post_filter", "connected_components_dedup"):
            exec(textwrap.dedent(ast.get_source_segment(src, node)), ns)
    graphs, E, P = postfilter_inputs()
    out["connected_components"] = [sorted(map(sorted, ns["connected_components"](None, neighbours(A)))) for A in graphs]
    out["get_violent_items"] = [int(v) for v in ns["get_violent_items"](None, P, E)]

    X = index_contract_rows()
    index = types.SimpleNamespace(search_and_reconstruct=lambda q, k: knn_ref.flat_search_and_reconstruct(X, q, k))
    svc = types.SimpleNamespace(get_non_uniques=lambda emb, threshold=0.94: R.get_non_uniques(emb, threshold))
    svc.connected_components_dedup = lambda emb: ns["connected_components_dedup"](svc, emb)
    svc.post_filter = lambda *a: ns["post_filter"](svc, *a)
    res = types.SimpleNamespace(image_index=index, text_index=index, metadata_is_ordered_by_ivf=False, safety_model=None,
                                violence_detector=None)
    q = X[3:4].astype(np.float32)
    for name, dedup in (("knn_search", False), ("knn_search_dedup", True)):
        dist, ind = ns["knn_search"](svc, q, "image", 40, res, dedup, False, False)
        out[name] = {"dist": [float(v) for v in dist], "ind": [int(v) for v in ind]}

    msrc = open(os.path.join(ref, "clip_retrieval", "clip_inference", "mapper.py")).read()
    mcls = next(n for n in ast.parse(msrc).body if isinstance(n, ast.ClassDef) and n.name == "ClipMapper")
    call = next(n for n in mcls.body if isinstance(n, ast.FunctionDef) and n.name == "__call__")
    mns = {"torch": torch, "np": np}
    exec(textwrap.dedent(ast.get_source_segment(msrc, call)), mns)
    fi, ft = mapper_features()
    me = types.SimpleNamespace(enable_image=True, enable_text=True, enable_metadata=True, use_mclip=False, device="cpu",
                               model_img=lambda x: fi.clone(), model_txt=lambda x: ft.clone())
    item = {"image_tensor": torch.zeros(5, 3, 4, 4), "text_tokens": torch.zeros(5, 77, dtype=torch.int64),
            "image_filename": list("abcde"), "text": list("vwxyz"), "metadata": list("12345")}
    r = mns["__call__"](me, item)
    out["mapper_call"] = {"keys": list(r), "image_embs": r["image_embs"].astype(np.float32).tolist(),
                          "text_embs": r["text_embs"].astype(np.float32).tolist(), "dtype": str(r["image_embs"].dtype),
                          "image_filename": r["image_filename"], "text": r["text"], "metadata": r["metadata"]}

    fx = {}
    for f in sorted(glob.glob(os.path.join(ref, "tests", "test_clip_inference", "test_tensors", "*.pkl"))):
        with open(f, "rb") as fh:
            o = pickle.load(fh)
        for name, t in zip(o["image_filename"], o["image_tensor"]):
            fx[name] = hashlib.sha256(t.numpy().astype(np.float32).tobytes()).hexdigest()
    out["preprocess_fixture_sha256"] = fx
    with open(os.path.join(HERE, "reference_calls.json"), "w") as fh:
        json.dump(out, fh, indent=0)


if __name__ == "__main__":
    main(sys.argv[1])
