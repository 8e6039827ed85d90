"""Both CLIP towers of every case of tower_ref.py (one per distinct architecture and activation of model.ARCHS, two
blocks per tower), under both weight sets of tower_ref.WEIGHTS, on the GPU against the float64 storage-emulating oracle
under its rounding envelope: raw fp32 features within 2 E of y_RN per row, normalised fp16 rows within the bound of
tower_ref.normalised_ratio.

What the kernel tests cannot see and these do: how clip_model.cu composes the kernels (the activation it picks, the
causal flag, leading dimensions, residual pointers and the positional row map of the patch GEMM, ln_pre in place, the
pooled row, the order of the layer), the chunk loop of encode_device, the captured-graph path of small batches, the
host entry's staging ring, and the persistent 128x256 GEMM that large batches take.  The oracle runs in float64 on the
same GPU.  Each (case, weight set) holds its handles and device weights only while its tests run."""
import functools

import numpy as np
import pytest
import torch

import tower_ref as R

pytestmark = pytest.mark.gpu

CASES = [(n, w) for n in R.cases() for w in R.WEIGHTS]
SEAM_MB = 2                 # chunks of 2 samples: a batch of 5 has seams after samples 1 and 3
SEAM_B = SEAM_MB + 3
WIDE_B = 40                 # every case's qkv GEMM takes the 128x256 kernel at 40 samples (checked below)


class Case:
    """One (case, weight set): its handles by max_batch, the oracle's device weights, the envelopes by sample, and the
    worst ratio to the bound of each check."""

    def __init__(self, name, weights):
        self.name, self.weights = name, weights
        self.label = "%s/%s" % (name, weights)
        self.arch = R.cases()[name]
        self.sd = R.state_dict(name, weights)
        self.W = R.handle_weights(self.sd, "cuda")
        self.models = {}
        self.worst = {}

    def model(self, max_batch):
        import clip_retrieval_b200 as m

        if max_batch not in self.models:
            self.models[max_batch] = m.B200Clip(self.arch, device=0, max_batch=max_batch).load_state_dict(self.sd)
        return self.models[max_batch]

    @functools.lru_cache(maxsize=None)
    def envelope(self, tower, i):
        return R.envelope(self.W, self.arch, tower, R.sample(self.arch, tower, i).cuda())

    def check(self, tower, what, rows, raw=None, norm=None):
        """raw [B, D] fp32 and / or norm [B, D] normalised rows of the batch that holds samples rows[0] .. rows[-1] at
        positions 0 .. len(rows)-1; every row inside its bound."""
        for k, i in enumerate(rows):
            y, E = self.envelope(tower, i)
            for kind, out, ratio in (("raw", raw, R.feature_ratio), ("norm", norm, R.normalised_ratio)):
                if out is None:
                    continue
                assert torch.isfinite(out[k].float()).all(), "%s %s %s sample %d: non-finite output" % (
                    self.label, tower, what, i)
                r = ratio(out[k], y, E)
                key = "%s %s %s" % (tower, what, kind)
                self.worst[key] = max(self.worst.get(key, 0.0), r)
                assert r <= 1.0, "%s %s %s sample %d: %s output at %.2f of the bound" % (
                    self.label, tower, what, i, kind, r)

    def report(self):
        for what, r in sorted(self.worst.items()):
            print("\n%-37s %-24s worst ratio %.3f" % (self.label, what, r))


@pytest.fixture(scope="module", params=CASES, ids=["%s-%s" % c for c in CASES])
def case(request):
    c = Case(*request.param)
    yield c
    c.report()
    c.envelope.cache_clear()
    del c.models, c.W
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _encode(model, tower, x):
    return model.encode_image(x) if tower == "image" else model.encode_text(x)


def _embed_device(model, tower, x):
    return model.embed_image_device(x) if tower == "image" else model.embed_text_device(x)


def _embed_host(model, tower, x):
    return model.embed_image(x) if tower == "image" else model.embed_text(x)


@pytest.mark.timeout(600)
def test_batch1_graph_path(case):
    """Batch 1 three times (eager, capture, replay): bit-identical, and inside the bound, raw and normalised."""
    arch = case.arch
    model = case.model(SEAM_MB)
    for tower in ("image", "text"):
        x = R.batch(arch, tower, 1).cuda()
        for call, what in ((_encode, "batch-1 graph"), (_embed_device, "batch-1 graph")):
            outs = [call(model, tower, x) for _ in range(3)]
            torch.cuda.synchronize()
            assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2]), \
                "%s %s: eager, captured and replayed forwards differ" % (case.label, tower)
            if call is _encode:
                case.check(tower, what, [0], raw=outs[0])
            else:
                case.check(tower, what, [0], norm=outs[0])


@pytest.mark.timeout(600)
def test_chunk_seams_and_entries(case):
    """max_batch + 3 samples through chunks of max_batch = 2: every sample (both sides of each seam) inside the bound;
    the host entry (staging ring) bit-identical to the device entry."""
    arch = case.arch
    model = case.model(SEAM_MB)
    rows = list(range(SEAM_B))
    for tower in ("image", "text"):
        x = R.batch(arch, tower, SEAM_B)
        raw = _encode(model, tower, x.cuda())
        norm = _embed_device(model, tower, x.cuda())
        host = _embed_host(model, tower, x)
        torch.cuda.synchronize()
        assert np.array_equal(host, norm.cpu().numpy()), "%s %s: host and device entries differ" % (case.label, tower)
        case.check(tower, "chunk seams", rows, raw=raw, norm=norm)


@pytest.mark.timeout(600)
def test_large_batch_wide_gemm(case):
    """WIDE_B samples in one chunk, where the persistent 128x256 GEMM runs: the first, a middle and the last sample
    inside the bound; host and device entries bit-identical."""
    from test_gemm_wide_gpu import pick_is_wide

    arch = case.arch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    model = case.model(WIDE_B)
    rows = [0, WIDE_B // 2, WIDE_B - 1]
    for tower in ("image", "text"):
        t, T = (arch.vision, R.image_tokens(arch)) if tower == "image" else (arch.text, arch.context_length)
        assert pick_is_wide(WIDE_B * T, 3 * t.width, sms), "%s %s: the qkv GEMM is not on the 128x256 kernel" % (
            case.label, tower)
        x = R.batch(arch, tower, WIDE_B)
        raw = _encode(model, tower, x.cuda())
        norm = _embed_device(model, tower, x.cuda())
        host = _embed_host(model, tower, x)
        torch.cuda.synchronize()
        assert np.array_equal(host, norm.cpu().numpy()), "%s %s: host and device entries differ" % (case.label, tower)
        case.check(tower, "large batch", [0], raw=raw[0:1], norm=norm[0:1])
        case.check(tower, "large batch", rows[1:2], raw=raw[rows[1]:rows[1] + 1], norm=norm[rows[1]:rows[1] + 1])
        case.check(tower, "large batch", rows[2:], raw=raw[rows[2]:], norm=norm[rows[2]:])
