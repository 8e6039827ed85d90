"""The query path of `clip-retrieval back` on the GPU (BASELINE configs[4]): a `KnnService`-compatible object.

Reference: `KnnService` (clip_retrieval/clip_back.py:200-470) — `query()` :419-470 = `compute_query` :207-255
(tokenise, `model.encode_text` / `encode_image` at batch 1, L2-normalise, fp32) -> `knn_search` :343-399
(`index.search_and_reconstruct(query, num_result_ids)` :362, -1 truncation :370-378, re-normalise :379,
`post_filter` :326-341 = dedup + violence prompts + safety model) -> `map_to_metadata` :401-417.
Here the query embedding never leaves the device between the text tower and the index scan, the reconstructed
rows stay in HBM for the post-filters, and only the surviving (id, similarity) pairs cross to the host.
`metadata_provider.get(ids, columns)` (clip_back.py:404-405) stays the caller's object (out of scope, SURVEY §2).

`MicroBatcher` is the batched request front of SURVEY §8(f) rank 4 (README.md:418: "for high throughput, using a
grpc server is required"): concurrent single queries are gathered for at most `max_wait_ms` into ONE text-tower
forward and ONE index pass — the nq >> 1 shape where the tensor-core scan wins.
"""
import threading
import time
from concurrent.futures import Future

import numpy as np


class ClipResource:
    """The fields of clip_back.ClipResource (clip_back.py:771-790) the query path reads."""

    def __init__(self, model, tokenizer=None, preprocess=None, image_index=None, text_index=None, device=None,
                 metadata_provider=None, columns_to_return=None, safety_model=None, violence_detector=None,
                 aesthetic_embeddings=None, ivf_old_to_new_mapping=None, model_txt_mclip=None):
        self.model = model
        self.model_txt_mclip = model_txt_mclip   # mclip.load_mclip(...) for use_mclip queries, or None
        self.tokenizer = tokenizer
        self.preprocess = preprocess
        self.image_index = image_index
        self.text_index = text_index
        self.device = device if device is not None else getattr(model, "device", "cuda")
        self.metadata_provider = metadata_provider
        self.columns_to_return = columns_to_return or []
        self.safety_model = safety_model
        self.violence_detector = violence_detector
        self.aesthetic_embeddings = aesthetic_embeddings
        self.ivf_old_to_new_mapping = ivf_old_to_new_mapping
        self.metadata_is_ordered_by_ivf = ivf_old_to_new_mapping is not None


class B200KnnService:
    """Same public methods and argument meaning as the reference's KnnService (minus the Flask plumbing)."""

    def __init__(self, clip_resources):
        self.clip_resources = clip_resources

    # ---- compute_query (clip_back.py:207-255) -------------------------------------------------------
    def compute_query_device(self, clip_resource, text_input=None, image_input=None, embedding_input=None,
                             text_tokens=None, aesthetic_score=None, aesthetic_weight=None, use_mclip=False,
                             mclip_tokens=None):
        """Normalised fp32 query [n, D] as a CUDA tensor.  `text_tokens` (int [n, 77]) bypasses the tokenizer
        (benchmarks: no BPE vocabulary exists offline); `image_input` is a PIL image or a preprocessed tensor.
        `use_mclip`: the text goes through `clip_resource.model_txt_mclip` (clip_back.py:222-224); `mclip_tokens` =
        (ids [n, T], lengths [n]) bypasses its tokenizer."""
        import torch

        model = clip_resource.model
        if use_mclip and (mclip_tokens is not None or (text_input is not None and text_input != "")):
            if clip_resource.model_txt_mclip is None:
                raise ValueError("use_mclip=True but this ClipResource has no model_txt_mclip "
                                 "(ClipResource(..., model_txt_mclip=load_mclip(clip_model)))")
            texts = None if mclip_tokens is not None else ([text_input] if isinstance(text_input, str) else list(text_input))
            q = clip_resource.model_txt_mclip.embed_device(texts, mclip_tokens)
        elif text_tokens is not None or (text_input is not None and text_input != ""):
            if text_tokens is None:
                text_tokens = clip_resource.tokenizer([text_input] if isinstance(text_input, str) else list(text_input))
            q = model.embed_text_device(torch.as_tensor(text_tokens).to(model.device), dtype=torch.float32)
        elif image_input is not None:
            if not isinstance(image_input, torch.Tensor):
                image_input = clip_resource.preprocess(image_input).unsqueeze(0)
            if image_input.dim() == 3:
                image_input = image_input.unsqueeze(0)
            q = model.embed_image_device(image_input.to(model.device), dtype=torch.float32)
        elif embedding_input is not None:
            q = torch.as_tensor(np.asarray(embedding_input, dtype=np.float32)).to(model.device)
            if q.dim() == 1:
                q = q.unsqueeze(0)
        else:
            raise ValueError("must fill one of text, image and image url input")
        if clip_resource.aesthetic_embeddings is not None and aesthetic_score is not None:
            a = torch.as_tensor(np.asarray(clip_resource.aesthetic_embeddings[aesthetic_score], dtype=np.float32)).to(q.device)
            q = q + a * float(aesthetic_weight)
            q = q / q.norm(dim=-1, keepdim=True)
        return q.contiguous()

    def compute_query(self, clip_resource, text_input, image_input, image_url_input, embedding_input, use_mclip,
                      aesthetic_score, aesthetic_weight):
        if image_url_input is not None and image_input is None and (text_input is None or text_input == ""):
            raise NotImplementedError("image_url input needs network access (download_image, clip_back.py:238-239)")
        return self.compute_query_device(clip_resource, text_input, image_input, embedding_input,
                                         aesthetic_score=aesthetic_score, aesthetic_weight=aesthetic_weight,
                                         use_mclip=use_mclip).cpu().numpy()

    # ---- post_filter (clip_back.py:326-341) on the device ----------------------------------------------
    def post_filter_device(self, safety_model, embeddings, deduplicate, use_safety_model, use_violence_detector,
                           violence_detector):
        """uint8 CUDA mask over the rows of `embeddings` (CUDA fp32 [n, d]): 1 = remove."""
        import torch
        from .postfilter import dedup_mask, get_unsafe_items, get_violent_items

        n = embeddings.shape[0]
        drop = torch.zeros(n, dtype=torch.uint8, device=embeddings.device)
        if n == 0:
            return drop
        if deduplicate:
            drop |= dedup_mask(embeddings)
        if use_violence_detector and violence_detector is not None:
            v = get_violent_items(violence_detector, embeddings)
            if len(v):
                drop[torch.as_tensor(v, device=drop.device, dtype=torch.long)] = 1
        if use_safety_model and safety_model is not None:
            u = get_unsafe_items(safety_model, embeddings)
            if len(u):
                drop[torch.as_tensor(u, device=drop.device, dtype=torch.long)] = 1
        return drop

    # ---- knn_search (clip_back.py:343-399) ---------------------------------------------------------------
    def knn_search(self, query, modality, num_result_ids, clip_resource, deduplicate, use_safety_model, use_violence_detector):
        import torch

        index = clip_resource.image_index if modality == "image" else clip_resource.text_index
        q = query if isinstance(query, torch.Tensor) else torch.as_tensor(np.ascontiguousarray(query, dtype=np.float32))
        q = q.to(clip_resource.model.device if clip_resource.model is not None else "cuda").contiguous()
        previous_nprobe = None
        if clip_resource.metadata_is_ordered_by_ivf and hasattr(index, "nprobe") and num_result_ids >= 100000:
            import math

            previous_nprobe = index.nprobe                       # clip_back.py:357-361
            index.nprobe = math.ceil(num_result_ids / 3000)
        try:
            need_rows = deduplicate or use_safety_model or use_violence_detector
            if need_rows and hasattr(index, "search_device"):
                try:
                    distances, indices, embeddings = index.search_device(q, num_result_ids, reconstruct=True)
                except TypeError:                                     # sharded wrappers return ids only
                    distances, indices = index.search_device(q, num_result_ids)
                    embeddings = None
            else:
                distances, indices = index.search_device(q, num_result_ids)
                embeddings = None
        finally:
            if previous_nprobe is not None:
                index.nprobe = previous_nprobe                         # clip_back.py:368-369
        ids, dist = indices[0], distances[0]
        nb = int((ids >= 0).sum().item()) if (ids < 0).any() else ids.numel()   # first -1 ends the list (:370-375)
        ids, dist = ids[:nb], dist[:nb]
        keep = torch.ones(nb, dtype=torch.bool, device=ids.device)
        if embeddings is not None and nb > 0:
            rows = embeddings[0][:nb]
            norms = rows.norm(dim=-1, keepdim=True)
            rows = rows / torch.where(norms == 0, torch.ones_like(norms), norms)          # normalized(), :193-197
            drop = self.post_filter_device(clip_resource.safety_model, rows, deduplicate, use_safety_model,
                                           use_violence_detector, clip_resource.violence_detector)
            keep &= drop == 0
        ids_h, dist_h, keep_h = ids.cpu().numpy(), dist.cpu().numpy(), keep.cpu().numpy()
        if clip_resource.metadata_is_ordered_by_ivf:
            ids_h = np.take(clip_resource.ivf_old_to_new_mapping, ids_h)
        # the reference also drops a result id it has already emitted or that a removed row carried (:388-397)
        removed = set(ids_h[~keep_h].tolist())
        out_i, out_d = [], []
        for ind, distance in zip(ids_h, dist_h):
            if ind not in removed:
                removed.add(ind)
                out_i.append(ind)
                out_d.append(distance)
        return out_d, out_i

    # ---- map_to_metadata (clip_back.py:401-417) -----------------------------------------------------------
    def map_to_metadata(self, indices, distances, num_images, metadata_provider, columns_to_return):
        metas = metadata_provider.get(indices[:num_images], columns_to_return) if metadata_provider is not None else []
        results = []
        for key, (d, i) in enumerate(zip(distances, indices)):
            output = {}
            meta = None if key + 1 > len(metas) else metas[key]
            if meta is not None:
                output.update(dict(meta))
            output["id"] = int(i)
            output["similarity"] = float(d)
            results.append(output)
        return results

    # ---- query (clip_back.py:419-470) ----------------------------------------------------------------------
    def query(self, text_input=None, image_input=None, image_url_input=None, embedding_input=None, modality="image",
              num_images=100, num_result_ids=100, indice_name=None, use_mclip=False, deduplicate=True,
              use_safety_model=False, use_violence_detector=False, aesthetic_score=None, aesthetic_weight=None,
              text_tokens=None, mclip_tokens=None):
        if (text_input is None and image_input is None and image_url_input is None and embedding_input is None
                and text_tokens is None and mclip_tokens is None):
            raise ValueError("must fill one of text, image and image url input")
        if indice_name is None:
            indice_name = next(iter(self.clip_resources.keys()))
        clip_resource = self.clip_resources[indice_name]
        query = self.compute_query_device(clip_resource, text_input, image_input, embedding_input, text_tokens,
                                          aesthetic_score, aesthetic_weight, use_mclip, mclip_tokens)
        distances, indices = self.knn_search(query, modality=modality, num_result_ids=num_result_ids,
                                             clip_resource=clip_resource, deduplicate=deduplicate,
                                             use_safety_model=use_safety_model, use_violence_detector=use_violence_detector)
        if len(distances) == 0:
            return []
        return self.map_to_metadata(indices, distances, num_images, clip_resource.metadata_provider,
                                    clip_resource.columns_to_return)


class MicroBatcher:
    """Gathers concurrent text queries into one forward + one index pass.

    `submit(text_tokens_row, k)` returns a Future of (distances [k], ids [k]) numpy arrays.  A worker thread takes
    whatever is queued (up to `max_batch`), waiting at most `max_wait_ms` after the first request of a batch —
    so a lone request pays at most that delay and a burst is served at the batched rate.  One worker per GPU
    process; under torchrun every rank must feed the same requests (queries are replicated, SURVEY §8e)."""

    def __init__(self, model, index, max_batch=64, max_wait_ms=0.2, k=40):
        self.model, self.index = model, index
        self.max_batch, self.max_wait = int(max_batch), float(max_wait_ms) / 1e3
        self.k = int(k)
        self._q = []
        self._cv = threading.Condition()
        self._stop = False
        self.batches = 0
        self.served = 0
        self._t = threading.Thread(target=self._run, daemon=True)
        self._t.start()

    def submit(self, tokens_row):
        f = Future()
        with self._cv:
            self._q.append((tokens_row, f))
            self._cv.notify()
        return f

    def close(self):
        with self._cv:
            self._stop = True
            self._cv.notify()
        self._t.join()

    def _run(self):
        import torch

        dev = self.model.device
        torch.cuda.set_device(dev)
        stream = torch.cuda.Stream(device=dev)
        while True:
            with self._cv:
                while not self._q and not self._stop:
                    self._cv.wait()
                if self._stop and not self._q:
                    return
                t0 = time.perf_counter()
                while len(self._q) < self.max_batch and not self._stop:
                    left = self.max_wait - (time.perf_counter() - t0)
                    if left <= 0:
                        break
                    self._cv.wait(left)
                batch, self._q = self._q[:self.max_batch], self._q[self.max_batch:]
            try:
                toks = torch.stack([torch.as_tensor(t) for t, _ in batch]).to(torch.int64)
                with torch.cuda.stream(stream):
                    q = self.model.embed_text_device(toks.to(dev, non_blocking=True), dtype=torch.float32)
                    D, I = self.index.search_device(q, self.k)
                    Dh, Ih = D.cpu().numpy(), I.cpu().numpy()
                for j, (_, f) in enumerate(batch):
                    f.set_result((Dh[j], Ih[j]))
            except Exception as e:  # noqa: BLE001 - delivered to the callers
                for _, f in batch:
                    if not f.done():
                        f.set_exception(e)
            self.batches += 1
            self.served += len(batch)
