"""The hit-shading instantiation ledger (texture_cases.HIT_SHADING) lists exactly the instantiations the launch sites select.

The launch sites are the `k_...<...><<<` lines of rt_shade.cu, gbuffer.cu and reference.cu, plus selections through a function pointer
(reference.cu's `kind == PASS_AO ? k_reference_mask<1> : k_reference_mask<0>`).  An instantiation added without naming the test that
compares it with the oracle fails here, on the CPU."""
import os

import texture_cases as TC

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "hybrid-rendering_b200", "csrc")
FILES = ("rt_shade.cu", "gbuffer.cu", "reference.cu")


def launched_instantiations(src):
    """instantiations of the hit-shading kernels named at launch sites in `src`, comments left out"""
    return TC.instantiations("\n".join(line.split("//")[0] for line in src.splitlines()))


def test_ledger_lists_exactly_the_launched_instantiations():
    found = set()
    for f in FILES:
        with open(os.path.join(CSRC, f)) as fh:
            found |= launched_instantiations(fh.read())
    assert len(found) == 20, sorted(found)
    assert set(TC.HIT_SHADING) == found, f"not in the ledger: {sorted(found - set(TC.HIT_SHADING))}; not launched: {sorted(set(TC.HIT_SHADING) - found)}"
    for inst, case in TC.HIT_SHADING.items():
        mod, test = case.split("::")
        assert os.path.exists(os.path.join(os.path.dirname(os.path.abspath(__file__)), mod)), case
        with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), mod)) as fh:
            assert f"def {test.split('[')[0]}(" in fh.read(), case
        if "[" in test:
            param = test.split("[")[1].rstrip("]")
            assert param in TC.CASES, case
            assert TC.textured(inst) == (param != "untextured"), inst


def test_parser_sees_launches_and_function_pointers():
    src = """
    if (x) k_path_trace<true, false><<<grid, 64, 0, st>>>(a);
    const auto k = kind == PASS_AO ? k_reference_mask<1> : k_reference_mask<0>;
    // k_gbuffer_render<true><<<  in a comment is not a launch
    k_reference_resolve<1><<<grid, 256>>>(g);
    """
    assert launched_instantiations(src) == {"k_path_trace<true, false>", "k_reference_mask<1>", "k_reference_mask<0>"}
