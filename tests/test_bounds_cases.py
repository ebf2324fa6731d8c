"""CPU: the case list of the memory-bounds tests (bounds_cases.py) is complete.  Every export that writes device memory has cases
or a reason to be left out, the list reaches every instance the host-side mirrors can select and every row-count edge, every
case is one the library accepts, and every case is needed: dropping one loses an instance or an edge."""
import numpy as np
import pytest
import torch

import bounds_cases as B
import dispatch_table as D
from bitblas_b200 import _lib


def test_every_writing_export_has_cases_or_a_reason():
    covered, excluded = B.entries(), set(B.EXCLUDED)
    assert not covered & excluded, covered & excluded
    missing = set(_lib.EXPORTS) - covered - excluded
    assert not missing, f"exports with neither a bounds case nor a reason in bounds_cases.EXCLUDED: {sorted(missing)}"
    assert covered | excluded <= set(_lib.EXPORTS), (covered | excluded) - set(_lib.EXPORTS)


def test_the_list_reaches_every_instance_and_edge():
    reached = set().union(*(B.labels(c) for c in B.CASES))
    missing = B.required() - reached
    assert not missing, f"not reached: {sorted(missing)}"


def test_every_case_is_needed():
    req = B.required()
    per = [B.labels(c) & req for c in B.CASES]
    for i, c in enumerate(B.CASES):
        others = set().union(*(p for j, p in enumerate(per) if j != i))
        assert per[i] - others, f"case {i} reaches nothing the others do not: {c}"


def _desc(c):
    int8 = c["A"] == "int8"
    fmt, bits = ("int" if c["W"].startswith("int") else "uint"), int(c["W"][-1])
    il = D.L_IL8 if int8 and c["il"] else (D.L_IL16 if c["il"] and not int8 else D.L_COMP)
    return D.desc(N=c["N"], K=c["K"], a_dtype={"float16": D.F16, "bfloat16": D.BF16, "int8": D.I8}[c["A"]],
                  w_fmt=D.W_INT if fmt == "int" else D.W_UINT, w_bits=bits, accum_dtype=D.I32 if int8 else D.F32,
                  out_dtype={"float16": D.F16, "bfloat16": D.BF16, "float32": D.F32, "int8": D.I8, "int32": D.I32}[c["out"]],
                  group_size=c["g"], with_scaling=int(c["mode"] != "none"),
                  with_zeros=int(c["mode"] in ("original", "rescale", "quantized")),
                  zeros_mode={"original": 0, "rescale": 1, "quantized": 2}.get(c["mode"], 0), with_bias=int(c["bias"]), w_layout=il,
                  w_tile=D.T_SLAB if c["tiled"] else D.T_ROW)


@pytest.mark.parametrize("i", range(len(B.MATMUL)))
def test_matmul_case_is_accepted_by_its_family(i):
    c = B.MATMUL[i]
    d = _desc(c)
    kid = B.FAMILY[c["family"]]["kid"]
    assert int(D.select(d, c["m"], kid)) == kid, (c, D.explain(d, c["m"]))
    if c["family"].startswith("gemm_ts"):
        kb = 128 if c["A"] == "int8" else 64
        assert int(D.ts_splits(d, c["m"], c["cap"] or B.FULL_SMS)) == c.get("split", 1), c
        assert c["K"] // kb % 2 == 1 or c.get("split") or c["tiled"], "an odd number of k-blocks"


def test_split_cases_split_only_at_their_cap():
    for c in B.MATMUL:
        if c.get("split"):
            assert c["cap"] == B.SPLIT_CAP


def test_slab_caps_end_a_range_inside_a_row_block():
    import exact_inputs as X
    props = [X.slab_coverage(c["N"], c["K"], c["cap"]) for c in B.MATMUL if c.get("prop")]
    assert any("range_inside_block" in p for p in props) and any("owner_stops_mid_block" in p for p in props)


def test_grouped_routings_pick_their_bucket():
    for e, routings in B.GROUPED_ROUTINGS.items():
        for name, counts in routings.items():
            if name.startswith(("nt", "bm")):
                assert B.grouped_bucket(e, counts) == name, (e, name)
    assert len(B.GROUPED_ROUTINGS["bb_matmul_grouped"]["e256"]) == 256


def test_guarded_layout_and_checks():
    g = B.Guarded(100, offset=16, fill=B.FILL["float16"], device="cpu")
    assert g.start % 256 == 16 and g.start >= B.MIN_GUARD and g.buf.numel() - g.start - g.nbytes >= B.MIN_GUARD
    g.seal()
    g.check_guards("fresh")
    g.payload()[:] = 0
    g.check_guards("payload written")
    with pytest.raises(AssertionError, match="an input was written"):
        g.check_unchanged("payload written")
    g.buf[g.start + g.nbytes] = 1
    with pytest.raises(AssertionError, match="back guard changed; first at payload end \\+0"):
        g.check_guards("one byte past the end")
    o = B.Guarded.output((3, 4), torch.float16, "float16", device="cpu")
    o.seal()
    o.view()[1, 2] = 0
    keep = torch.zeros(3, 4, dtype=torch.bool)
    o.check_kept(keep, "nothing kept")
    keep[1] = True
    with pytest.raises(AssertionError, match="unwritten were written; first at \\[\\[1, 2\\]\\]"):
        o.check_kept(keep, "row 1 kept")
    assert B.guard_for(4096) == 128 * 4096 and B.guard_for(1) == B.MIN_GUARD
    assert np.frombuffer(B.OUT_FILL["float16"], np.float16).item() != np.frombuffer(B.OUT_FILL["float16"], np.float16).item()
