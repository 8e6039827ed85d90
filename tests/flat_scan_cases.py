"""Case table of the flat exhaustive scan (csrc/knn_scan.cu, csrc/knn_mma.cu) and the kernel instantiations it
must reach.  Imported by tests/test_flat_scan_gpu.py, which runs every case and asserts the plan the library
reports (`last_scan_plan()`), and by tests/test_flat_scan_table_cpu.py, which checks without a GPU that the
table reaches every instantiation.  A change to `plan_scan` that moves a case to another kernel fails that case
by name; one that drops an instantiation from the table fails the CPU check.
"""

REGISTER, STAGED, SPLIT, HI_ONLY = 0, 1, 2, 3   # `kernel` of b200_index_last_scan_plan

# set_tensor_scan flags: 1 = wgmma scan on (default), 0 = FMA scan through the bulk-copy ring, 4 = register FMA scan
DEFAULT, FMA_RING, FMA_REGISTER = 1, 0, 4

# every template instantiation the dispatch can pick: (kernel, queries per pass NQ, chunks per lane CH)
INSTANTIATIONS = (
    {(STAGED, nq, ch) for nq in (1, 2) for ch in range(1, 5)}
    | {(STAGED, 4, ch) for ch in range(1, 4)}
    | {(REGISTER, 1, ch) for ch in range(1, 9)}
    | {(REGISTER, 2, ch) for ch in range(1, 7)}
    | {(REGISTER, 4, ch) for ch in range(1, 4)}
)
RANGE_INSTANTIATIONS = set(range(1, 9))   # range_scan_kernel<CH>


def ch_of(d):
    """16-byte chunks per lane: ceil(d / 256)."""
    return (d // 8 + 31) // 32


# Widths per CH: one that ends inside its last chunk (d % 256 != 0) and the full 256 * CH.  d = 8 is one chunk on
# lane 0 only, d = 264 a second chunk on lane 0 only, d = 2040 a last chunk on 31 lanes.
WIDTHS = (8, 200, 256, 264, 512, 520, 768, 776, 1024, 1032, 1280, 1288, 1536, 1544, 1792, 1800, 2040, 2048)
RANGE_WIDTHS = (8, 200, 264, 520, 776, 1032, 1288, 1544, 1800, 2040, 2048)

# Every instantiation, at every width of WIDTHS: (d, nq, flags) -> (kernel, NQ).  nq = 3 leaves the last pass of
# NQ = 2 half empty, nq = 7 the last pass of NQ = 4 (or of NQ = 2 when CH = 4..6) three quarters full.
# Register kernel: nq = 1 -> NQ 1; nq = 3 -> NQ 2 up to CH 6, NQ 1 above (NQ * CH <= 12); nq = 7 -> NQ 4 up to CH 3,
# NQ 2 up to CH 6.  Ring: NQ 1 and 2 up to CH 4, NQ 4 up to CH 3; at CH >= 5 nq <= 4 has only the register kernel.
_REG_NQ = {1: {1: 1, 3: 2, 7: 4}, 2: {1: 1, 3: 2, 7: 4}, 3: {1: 1, 3: 2, 7: 4}, 4: {1: 1, 3: 2, 7: 2},
           5: {1: 1, 3: 2, 7: 2}, 6: {1: 1, 3: 2, 7: 2}, 7: {1: 1, 3: 1}, 8: {1: 1, 3: 1}}
_RING_NQ = {1: {1: 1, 3: 2, 7: 4}, 2: {1: 1, 3: 2, 7: 4}, 3: {1: 1, 3: 2, 7: 4}, 4: {1: 1, 3: 2, 7: 2}}

INSTANTIATION_CASES = []   # (d, nq, flags, (kernel, NQ, CH))
for _d in WIDTHS:
    _ch = ch_of(_d)
    for _nq, _NQ in sorted(_REG_NQ[_ch].items()):
        INSTANTIATION_CASES.append((_d, _nq, FMA_REGISTER, (REGISTER, _NQ, _ch)))
    for _nq, _NQ in sorted(_RING_NQ.get(_ch, {}).items()):
        # nq > 4 with the default flags would take the wgmma scan
        INSTANTIATION_CASES.append((_d, _nq, DEFAULT if _nq <= 4 else FMA_RING, (STAGED, _NQ, _ch)))
    if _ch >= 5:
        INSTANTIATION_CASES.append((_d, 1, DEFAULT, (REGISTER, 1, _ch)))   # default flags: no ring kernel this wide

# Both sides of every switch of the dispatch: name -> [(d, nq, k, n, flags, (kernel, NQ, CH))].  The cases of one
# name must agree on ids with each other (where their float64 scores differ by more than 2 * TOL) and with float64.
BOUNDARY_CASES = {
    # tensor scan: nq > 4, k <= 128, n >= 4096, d >= 64
    "nq4-5": [(768, 4, 40, 38021, DEFAULT, (STAGED, 4, 3)), (768, 5, 40, 38021, DEFAULT, (SPLIT, 128, 3))],
    "k128-129": [(768, 5, 128, 38021, DEFAULT, (SPLIT, 128, 3)), (768, 5, 129, 38021, DEFAULT, (STAGED, 4, 3))],
    "n4095-4096": [(768, 5, 40, 4095, DEFAULT, (STAGED, 4, 3)), (768, 5, 40, 4096, DEFAULT, (SPLIT, 128, 3))],
    "d56-nq5": [(56, 5, 40, 38021, DEFAULT, (STAGED, 4, 1))],
    "d64-nq5": [(64, 5, 40, 38021, DEFAULT, (SPLIT, 128, 1))],
    "d72-nq5": [(72, 5, 40, 38021, DEFAULT, (SPLIT, 128, 1))],
    "d56-nq300": [(56, 300, 40, 38021, DEFAULT, (STAGED, 4, 1))],
    "d64-nq300": [(64, 300, 40, 38021, DEFAULT, (HI_ONLY, 256, 1))],
    "d72-nq300": [(72, 300, 40, 38021, DEFAULT, (HI_ONLY, 256, 1))],
    # queries per pass halve when NQ * k > 1536 (the per-warp lists of 8 warps in 96 KB)
    "nqk1536-ring": [(256, 4, 384, 38021, DEFAULT, (STAGED, 4, 1)), (256, 4, 385, 38021, DEFAULT, (STAGED, 2, 1))],
    "nqk1536-register": [(256, 4, 384, 38021, FMA_REGISTER, (REGISTER, 4, 1)),
                         (256, 4, 385, 38021, FMA_REGISTER, (REGISTER, 2, 1))],
    # the ring needs its lists + 256 B + 3 slots of 32 rows within 220 KB: at d = 1024, NQ = 2 that is k <= 222
    "ring-fallback": [(1024, 2, 222, 38021, DEFAULT, (STAGED, 2, 4)), (1024, 2, 223, 38021, DEFAULT, (REGISTER, 2, 4))],
    # the FMA path runs 64 queries per batch of candidate lists (k > 128 keeps it off the tensor scan)
    "qb64": [(256, 64, 129, 20011, DEFAULT, (STAGED, 4, 1)), (256, 65, 129, 20011, DEFAULT, (STAGED, 4, 1)),
             (256, 130, 129, 20011, DEFAULT, (STAGED, 4, 1))],
}

# k at the edges of a warp's list (31/32/33 lanes), 1 and the 8192 maximum: (d, nq, k, flags) -> (kernel, NQ, CH).
# At k = 8192 the lists of every NQ > 1 exceed 96 KB and the ring's do not fit at all: the register kernel, NQ = 1.
K_VALUES = (1, 31, 32, 33, 8192)
K_CASES = []
for _d, _flags, _kernel, _nqs in ((200, FMA_REGISTER, REGISTER, {1: 1, 2: 2, 4: 4}),
                                  (1288, FMA_REGISTER, REGISTER, {1: 1, 2: 2, 4: 2}),
                                  (200, DEFAULT, STAGED, {1: 1, 2: 2, 4: 4}),
                                  (776, DEFAULT, STAGED, {1: 1, 2: 2, 4: 2})):
    for _nq, _NQ in sorted(_nqs.items()):
        for _k in K_VALUES:
            K_CASES.append((_d, _nq, _k, _flags, (REGISTER, 1, ch_of(_d)) if _k == 8192 else (_kernel, _NQ, ch_of(_d))))


def all_plans():
    """Every (kernel, NQ, CH) the table expects."""
    plans = {p for _, _, _, p in INSTANTIATION_CASES}
    plans |= {c[-1] for cases in BOUNDARY_CASES.values() for c in cases}
    plans |= {p for _, _, _, _, p in K_CASES}
    return plans
