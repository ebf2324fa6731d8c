"""CPU: the library's kernel choice (bb_select_kernel, under every kernel override) and bb_workspace_bytes against the Python mirror
of the dispatch table (dispatch_table.py) on a grid of descriptors, and the boundary-class coverage of the GPU edge sweep's case list
(test_gpu_dispatch_edges.py).  Needs the built library, no GPU."""
from __future__ import annotations

import ctypes
import itertools

import numpy as np
import pytest
import torch

import dispatch_table as D

A_TYPES = [D.F16, D.BF16, D.I8]
W_TYPES = [(D.W_UINT, b) for b in (1, 2, 4, 8)] + [(D.W_INT, b) for b in (1, 2, 4, 8)] + \
          [(D.W_NF, 4), (D.W_FP4, 4), (D.W_E4M3, 8), (D.W_E5M2, 8)]
ACCUM = {D.F16: [D.F32, D.F16, D.BF16], D.BF16: [D.F32, D.BF16, D.F16], D.I8: [D.I32]}
OUT = {D.F16: [D.F16, D.BF16, D.F32], D.BF16: [D.BF16, D.F32, D.F16], D.I8: [D.I32, D.I8, D.F16, D.BF16, D.F32]}
# (with_scaling, with_zeros, zeros_mode); zeros without scaling (validate accepts it, no fast family does) takes every mode in turn
ZEROS = [(0, 0, 0), (1, 0, 0), (1, 1, D.Z_ORIGINAL), (1, 1, D.Z_RESCALE), (1, 1, D.Z_QUANTIZED), (0, 1, -1)]
GROUPS = [-1, 32, 64, 128, 192, 256, 320, 384, 512]
NS = [8, 16, 24, 48, 72, 112, 128, 144, 272, 400, 1376, 2368, 2752, 3696, 19200]
KS = [32, 64, 96, 192, 256, 576, 640, 768, 1280, 1376, 1536, 2048]
# every m of the grid is one of these; each valid descriptor is checked at one m of every class (the predicates' thresholds are
# m == 1, m <= 8, m <= 32; the split-K factor and the wgmma tile change at 32, 64 and 128)
M_CLASSES = [[1], list(range(2, 9)), list(range(9, 33)), [33, 64, 65, 128, 129, 300, 4096]]
M_ALL = sorted(set(itertools.chain(*M_CLASSES)))


def descriptor_grid():
    """the record array of every combination of A type, weight type, layout, tile and zeros mode with every (N, K, g); the
    accumulation type, output type and bias rotate with the index"""
    types = list(itertools.product(A_TYPES, W_TYPES, [D.L_COMP, D.L_IL16, D.L_IL8], [D.T_ROW, D.T_SLAB], ZEROS))
    shapes = list(itertools.product(NS, KS, GROUPS))
    rec = np.zeros(len(types) * len(shapes), dtype=D.record_dtype())
    t = np.repeat(np.arange(len(types)), len(shapes))
    s = np.tile(np.arange(len(shapes)), len(types))
    i = np.arange(rec.size)
    tt = np.array([(a, f, b, lay, tile, ws, wz, zm) for a, (f, b), lay, tile, (ws, wz, zm) in types], dtype=np.int64)[t]
    ss = np.array(shapes, dtype=np.int64)[s]
    rec["N"], rec["K"], rec["group_size"] = ss[:, 0], ss[:, 1], ss[:, 2]
    rec["a_dtype"], rec["w_fmt"], rec["w_bits"], rec["w_layout"], rec["w_tile"] = tt[:, 0], tt[:, 1], tt[:, 2], tt[:, 3], tt[:, 4]
    rec["with_scaling"], rec["with_zeros"] = tt[:, 5], tt[:, 6]
    rec["zeros_mode"] = np.where(tt[:, 7] < 0, i % 3, tt[:, 7])
    for a in A_TYPES:
        sel = tt[:, 0] == a
        rec["accum_dtype"][sel] = np.array(ACCUM[a])[i[sel] % len(ACCUM[a])]
        rec["out_dtype"][sel] = np.array(OUT[a])[(i[sel] // 7) % len(OUT[a])]
    rec["with_bias"] = (i // 3) % 2
    return rec


def m_slots(n):
    """[n, 4]: the m of each class for descriptor i (strides coprime to the class sizes, so every m meets every shape)"""
    i = np.arange(n, dtype=np.int64)
    strides = (1, 3, 5, 2)
    return np.stack([np.asarray(c, dtype=np.int64)[(i * s) % len(c)] for s, c in zip(strides, M_CLASSES)], 1)


def _sms():
    """the SM count the library sizes its work for: the device's, or its fallback of 132 (an H100 SXM) without a device"""
    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


@pytest.fixture(scope="module")
def lib():
    from bitblas_b200 import _lib
    lib = _lib.load()
    lib.bb_set_kernel_override(D.AUTO)
    yield lib
    lib.bb_set_kernel_override(D.AUTO)


def _raw(lib):
    """bb_select_kernel and bb_workspace_bytes taking the descriptor's address as an integer (the grid is one buffer)"""
    sel = ctypes.CFUNCTYPE(ctypes.c_int, ctypes.c_void_p, ctypes.c_int)(("bb_select_kernel", lib))
    ws = ctypes.CFUNCTYPE(ctypes.c_size_t, ctypes.c_void_p, ctypes.c_int)(("bb_workspace_bytes", lib))
    return sel, ws


def _report(rec, idx, m, override, got, want, what):
    lines = [f"{what}: {len(idx)} descriptors disagree with the mirror (override {D.NAME.get(override, override)})"]
    for j in idx[:5]:
        d = D.grid_view(rec[j:j + 1])
        one = D.SimpleNamespace(**{f: np.int64(getattr(d, f)[0]) for f in D.FIELDS})
        fields = ", ".join(f"{f}={int(getattr(one, f))}" for f in D.FIELDS)
        lines.append(f"  m={int(m[j])} {fields}: library {got[j]} mirror {want[j]}; first failing clause per predicate "
                     f"{D.explain(one, int(m[j]))}")
    return "\n".join(lines)


def test_library_dispatch_matches_the_mirror(lib, capsys):
    rec = descriptor_grid()
    base = rec.ctypes.data
    size = rec.dtype.itemsize
    sel, ws = _raw(lib)
    d = D.grid_view(rec)
    n = rec.size
    sms = _sms()
    valid = np.asarray(D.holds(D.VALIDATE_CLAUSES, d))
    vi = np.nonzero(valid)[0]
    vd = D.grid_view(rec[vi])
    slots = m_slots(vi.size)
    compared = 0
    # rejected descriptors: -1 at every m and under every override, no workspace
    inv = np.nonzero(~valid)[0]
    got = np.array([sel(base + int(j) * size, 1) for j in inv])
    bad = inv[got != -1]
    assert bad.size == 0, _report(rec, bad, np.ones(n, np.int64), D.AUTO, dict(zip(inv, got)), dict.fromkeys(inv, -1), "validate")
    assert all(ws(base + int(j) * size, 1) == 0 for j in inv[::97])
    compared += inv.size
    for s in range(slots.shape[1]):
        m = slots[:, s]
        want_k = D.select(vd, m)
        want_ws = D.workspace_bytes(vd, m, sms)
        got_k = np.array([sel(base + int(j) * size, int(mm)) for j, mm in zip(vi, m)])
        got_ws = np.array([ws(base + int(j) * size, int(mm)) for j, mm in zip(vi, m)], dtype=np.int64)
        mm_full = np.zeros(n, np.int64)
        mm_full[vi] = m
        bad = np.nonzero(got_k != want_k)[0]
        assert bad.size == 0, _report(rec, vi[bad], mm_full, D.AUTO, dict(zip(vi, got_k)), dict(zip(vi, want_k)), "bb_select_kernel")
        bad = np.nonzero(got_ws != want_ws)[0]
        assert bad.size == 0, _report(rec, vi[bad], mm_full, D.AUTO, dict(zip(vi, got_ws)), dict(zip(vi, want_ws)),
                                      "bb_workspace_bytes")
        compared += 2 * vi.size
    # every forced family at m = 1 and at the m of the third class (9 .. 32, where all four fast families can apply)
    try:
        for fam in D.FAMILIES:
            lib.bb_set_kernel_override(fam)
            for s in (0, 2):
                m = slots[:, s]
                want_k = D.select(vd, m, fam)
                got_k = np.array([sel(base + int(j) * size, int(mm)) for j, mm in zip(vi, m)])
                mm_full = np.zeros(n, np.int64)
                mm_full[vi] = m
                bad = np.nonzero(got_k != want_k)[0]
                assert bad.size == 0, _report(rec, vi[bad], mm_full, fam, dict(zip(vi, got_k)), dict(zip(vi, want_k)),
                                              f"bb_select_kernel forced to {D.NAME[fam]}")
                compared += vi.size
    finally:
        lib.bb_set_kernel_override(D.AUTO)
    # every family is reached somewhere on the grid under auto dispatch
    reached = set(np.unique(D.select(vd, slots[:, 0])).tolist()) | set(np.unique(D.select(vd, slots[:, 2])).tolist()) | \
        set(np.unique(D.select(vd, slots[:, 3])).tolist())
    assert reached >= set(D.FAMILIES), reached
    with capsys.disabled():
        print(f"\n[dispatch table] {n} descriptors ({vi.size} valid), {compared} (descriptor, m, override) points agree with "
              f"the mirror; SM count {sms}")


def test_grid_covers_the_listed_values():
    rec = descriptor_grid()
    d = D.grid_view(rec)
    assert set(np.unique(rec["N"])) == set(NS) and set(np.unique(rec["K"])) == set(KS)
    assert set(np.unique(rec["group_size"])) == set(GROUPS)
    valid = np.asarray(D.holds(D.VALIDATE_CLAUSES, d))
    m = m_slots(int(valid.sum()))
    assert set(np.unique(m)) == set(M_ALL)
    # every accepted (A, accum, out) triple, layout, tile and zeros mode, with and without bias, among the valid descriptors
    v = rec[valid]
    triples = set(zip(v["a_dtype"].tolist(), v["accum_dtype"].tolist(), v["out_dtype"].tolist()))
    assert triples == {(a, c, o) for a in A_TYPES for c in ACCUM[a] for o in OUT[a]}, triples
    for f in ("w_layout", "w_tile", "zeros_mode", "with_bias"):
        assert len(np.unique(v[f])) >= 2, f
    assert set(zip(v["w_fmt"].tolist(), v["w_bits"].tolist())) == set(W_TYPES)


def test_mirror_names_the_clause():
    """explain() names the clause that puts a descriptor on the rejecting side of each predicate"""
    d = D.desc(N=1376, K=1376, group_size=-1, w_layout=D.L_IL16)
    e = D.explain(d, 40)
    assert e["validate"] is None and e["gemm_ts_supported"] == "N % 128" and e["gemv_mma_supported"] == "1 <= m <= 32"
    assert D.explain(d, 1)["gemv_mma_supported"] == "K % 128" and D.explain(d, 1)["gemv_slab_supported"] == "K % 256"
    assert int(D.select(d, 40)) == D.GENERIC
    d = D.desc(N=3696, K=8192, group_size=128, with_scaling=1)
    assert int(D.select(d, 1)) == D.GEMV_SLAB and int(D.select(d, 16)) == D.GEMV_MMA and int(D.select(d, 16, D.GEMM_TS)) == -1
    assert D.explain(d, 1)["gemv_slab_supported"] is None and D.explain(d, 16)["gemm_ts_supported"] == "N % 128"
    d = D.desc(N=1376, K=4096, group_size=128, with_scaling=1)
    assert int(D.select(d, 16)) == D.GEMV_MMA and D.explain(d, 16)["gemm_ts_supported"] == "N % 128"
    assert int(D.select(d, 33)) == D.GENERIC
    assert D.explain(D.desc(K=1000, group_size=128), 1)["validate"] == "K % g"


# ---- the GPU sweep's case list ---------------------------------------------------------------------------------------------------
def test_edge_cases_reach_every_boundary_class(lib, capsys):
    import test_gpu_dispatch_edges as E
    hit = {}
    for c in E.CASES:
        for cls in E.classes_of(c, sms=132):
            hit.setdefault(cls, []).append(c["id"])
    missing = [c for c in E.BOUNDARY_CLASSES if c not in hit]
    with capsys.disabled():
        print(f"\n[dispatch edges] {len(E.CASES)} GPU cases reach {len(E.BOUNDARY_CLASSES) - len(missing)}/"
              f"{len(E.BOUNDARY_CLASSES)} boundary classes (at 132 SMs)")
        for cls in E.BOUNDARY_CLASSES:
            print(f"  {cls}: {len(hit.get(cls, []))} cases")
    assert not missing, f"boundary classes no case reaches: {missing}"


def test_edge_case_descriptors_are_the_operators(lib):
    """the descriptor the coverage test derives from each case is the one Matmul builds for it"""
    import test_gpu_dispatch_edges as E
    for c in E.CASES:
        op = E.operator_of(c)
        assert vars(D.from_struct(op._desc)) == vars(E.desc_of(c)), c["id"]
    assert len({c["id"] for c in E.CASES}) == len(E.CASES)
