"""The flat-scan case table (tests/flat_scan_cases.py) reaches every kernel instantiation of csrc/knn_scan.cu.
Runs without a GPU; tests/test_flat_scan_gpu.py runs the cases and asserts the plan of each."""
import os
import re

from flat_scan_cases import (BOUNDARY_CASES, INSTANTIATION_CASES, INSTANTIATIONS, K_CASES, RANGE_INSTANTIATIONS,
                             RANGE_WIDTHS, REGISTER, STAGED, all_plans, ch_of)

SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "clip-retrieval_b200", "csrc",
                   "knn_scan.cu")


def _body(src, signature):
    return re.search(re.escape(signature) + r" \{(.*?)\n\}", src, re.S).group(1)


def _dispatchable():
    """(kernel, NQ, CH) of every flat_scan_kernel / flat_scan_staged_kernel the pick_* functions of knn_scan.cu can
    return, and the CH of every range_scan_kernel pick_range can return."""
    src = open(SRC).read()
    found = set()
    for kernel, name, pick_nq, pick_ch in ((REGISTER, "flat_scan_kernel", "static scan_fn pick_scan(int nqp, int ch)",
                                            "static scan_fn pick_ch(int ch)"),
                                           (STAGED, "flat_scan_staged_kernel", "static staged_fn pick_staged(int nqp, int ch)",
                                            "static staged_fn pick_staged_ch(int ch)")):
        nqs = {int(v) for v in re.findall(r"pick_\w*ch<(\d+)>", _body(src, pick_nq))}
        assert nqs == {1, 2, 4}
        # the switch of pick_*_ch: unguarded cases first, then blocks guarded by `if constexpr (NQ <= n / == n)`
        for i, part in enumerate(_body(src, pick_ch).split("if constexpr")):
            chs = {int(c) for c in re.findall(name + r"<NQ, (\d+)>", part)}
            if i == 0:
                ok = nqs
            else:
                op, lim = re.match(r"\s*\(NQ (<=|==) (\d+)\)", part).groups()
                ok = {nq for nq in nqs if (nq <= int(lim) if op == "<=" else nq == int(lim))}
            found |= {(kernel, nq, ch) for nq in ok for ch in chs}
    ranges = {int(c) for c in re.findall(r"range_scan_kernel<(\d+)>", _body(src, "static range_fn pick_range(int ch)"))}
    return found, ranges


def test_table_reaches_every_instantiation():
    assert len([p for p in INSTANTIATIONS if p[0] == STAGED]) == 11
    assert len([p for p in INSTANTIATIONS if p[0] == REGISTER]) == 17
    missing = INSTANTIATIONS - {p for _, _, _, p in INSTANTIATION_CASES}
    assert not missing, "no case runs %s" % sorted(missing)
    assert {ch_of(d) for d in RANGE_WIDTHS} == RANGE_INSTANTIATIONS == set(range(1, 9))


def test_table_matches_the_dispatch_source():
    """The instantiation list is the one the dispatch can pick: a kernel added to or removed from a pick_* switch
    must be added to or removed from the table, with a case that runs it."""
    kernels, ranges = _dispatchable()
    assert kernels == INSTANTIATIONS
    assert ranges == RANGE_INSTANTIATIONS


def test_every_expected_plan_exists():
    """Each case expects an FMA instantiation that exists (or a tensor-core plan), at the CH of its width."""
    assert {p for p in all_plans() if p[0] in (REGISTER, STAGED)} <= INSTANTIATIONS
    for d, _, _, p in INSTANTIATION_CASES:
        assert p[2] == ch_of(d), (d, p)
    for name, cases in BOUNDARY_CASES.items():
        for d, _, _, _, _, p in cases:
            assert p[2] == ch_of(d), (name, d, p)
    for d, _, _, _, p in K_CASES:
        assert p[2] == ch_of(d), (d, p)
