"""Coverage guard of the element-wise kernel matrix (no GPU): every kernel, and every template instantiation, that
engine.cu's element-wise launchers can launch has a row in tests/test_elem_matrix_gpu.py's INSTANTIATIONS, and every row
names a case that expects it.  The launchers are parsed: the gn_apply_kernel<NOUT, RAW> instantiations of
launch_groupnorm, the layernorm_quant_kernel<NVEC> instantiations of launch_layernorm and every launch_k(qd::..._kernel
call.  Kernels that other matrices own (GEMM, quantised attention, sampler updates) are listed with the file that
tests them.  A kernel added to a launcher without a test fails here on a machine with no GPU."""
import os
import re

from tests import test_elem_matrix_gpu as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENGINE = os.path.join(ROOT, "q-diffusion_b200", "csrc", "engine.cu")


def _body(src, signature):
    m = re.search(r"\n" + re.escape(signature) + r" \{\n(.*?)\n\}\n", src, re.S)
    assert m, f"{signature} not found in engine.cu"
    return m.group(1)


def _launched():
    src = open(ENGINE).read()
    names = set(re.findall(r"launch_k\(qd::(\w+_kernel)\b", src))
    templated = {n for n in names if re.search(r"launch_k\(qd::" + n + r"<", src)}
    names -= templated
    gn = _body(src, "int launch_groupnorm(const qd_groupnorm_desc& d, cudaStream_t s)")
    apply = re.findall(r"QD_GN_APPLY\((\d+),\s*(true|false)\)", gn)
    assert apply, "no gn_apply_kernel instantiation found in launch_groupnorm"
    names |= {f"gn_apply_kernel<{n},{r}>" for n, r in apply}
    ln = _body(src, "int launch_layernorm(const qd_layernorm_desc& d, cudaStream_t s)")
    nvec = re.findall(r"launch_layernorm_t<(\d+)>", ln)
    assert nvec, "no layernorm_quant_kernel instantiation found in launch_layernorm"
    names |= {f"layernorm_quant_kernel<{v}>" for v in nvec}
    return names, templated


def test_templated_kernels_are_the_expanded_ones():
    _, templated = _launched()
    assert templated <= {"gn_apply_kernel", "layernorm_quant_kernel", "gemm_i8_kernel", "qattention_kernel",
                         "qattention_smallk_kernel", "qattention_wg_kernel", "att_krowsum_kernel"}, templated


def test_every_kernel_has_a_row():
    names, _ = _launched()
    names = {n for n in names if n.split("<")[0] not in E.OTHER_MATRICES}
    assert len(names) >= 35, sorted(names)
    assert set(E.INSTANTIATIONS) == names, (
        f"missing rows: {sorted(names - set(E.INSTANTIATIONS))}; rows without a launch: "
        f"{sorted(set(E.INSTANTIATIONS) - names)}")


def test_other_matrices_exist():
    src = open(ENGINE).read()
    for kernel, path in E.OTHER_MATRICES.items():
        assert re.search(r"qd::" + kernel + r"\b", src), kernel
        assert os.path.exists(os.path.join(ROOT, path)), path


def test_every_row_names_a_case_that_expects_it():
    for kernel, cid in E.INSTANTIATIONS.items():
        assert cid in E.CASES, (kernel, cid)
        assert kernel in E.CASES[cid]["expect"], (kernel, cid, sorted(E.CASES[cid]["expect"]))


def test_every_case_expects_known_kernels():
    for cid, c in E.CASES.items():
        assert c["expect"] and c["expect"] <= set(E.INSTANTIATIONS), (cid, sorted(c["expect"] - set(E.INSTANTIATIONS)))


def test_groupnorm_thresholds_are_straddled():
    """Each path-choice threshold of launch_groupnorm has a case on either side, and every gn_apply instantiation runs
    behind both the partial-sum and the GEMM-statistics passes."""
    gn = {cid: c for cid, c in E.CASES.items() if c["op"] == "groupnorm"}

    def units(c):
        return c["HW"] * (c["C"] // c["groups"] // 2)

    assert any(units(c) == 5120 and c["path"] == "fused" for c in gn.values())
    assert any(units(c) > 5120 and c["path"] == "partial" and c["C"] // c["groups"] == 2 for c in gn.values())
    assert any(c["B"] * c["groups"] == 2048 and c["path"] == "fused" for c in gn.values())
    assert any(c["B"] * c["groups"] > 2048 and c["path"] == "partial" and units(c) <= 5120 for c in gn.values())
    cpgs = {c["C"] // c["groups"] for c in gn.values()}
    assert {128, 130} <= cpgs and any(p % 2 for p in cpgs)
    for n_out in range(4):
        for raw in (False, True):
            for path in ("partial", "stats"):
                assert any(c["path"] == path and c["n_out"] == n_out and c["raw"] == raw for c in gn.values()), (n_out, raw, path)
    assert {c["kappa"] for c in gn.values()} >= {10, 100}


def test_layernorm_widths():
    want = {4, 128, 132, 320, 512, 640, 768, 1024, 1152, 1280, 1536, 2048}
    got = {c["C"] for c in E.CASES.values() if c["op"] == "layernorm"}
    assert want <= got, want - got
