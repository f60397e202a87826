"""CPU suite: the C-ABI library builds, loads and exports every symbol include/hyphy_b200.h declares;
without a GPU it fails loudly instead of falling back."""
import os
import re

import pytest

from hyphy_b200 import engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "hyphy_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(hb2_[a-z0-9_]+)\s*\(", text)))


def test_header_symbols_all_exported(engine_lib):
    declared = _declared_symbols()
    assert len(declared) >= 14
    for name in declared:
        assert hasattr(engine_lib, name), f"{name} declared in include/hyphy_b200.h but not exported"
    assert sorted(n for n, _, _ in engine.ABI) == declared


def test_abi_version(engine_lib):
    assert engine_lib.hb2_abi_version() == 1


def test_no_cpu_fallback(engine_lib):
    """No GPU => create must fail with an explicit message (the host treats it as fatal)."""
    if engine.device_count() > 0:
        pytest.skip("a GPU is visible here")
    from hyphy_b200 import synth, LikelihoodFunction, EngineError
    with pytest.raises(EngineError, match="no CPU fallback"):
        LikelihoodFunction(synth.nucleotide_workload(4, 10))


def test_create_refuses_fractional_ambiguity(engine_lib):
    """Ambiguity rows are 0/1 (the reference's resolution vectors); create refuses any other weight, GPU or not."""
    import dataclasses
    import numpy as np
    from hyphy_b200 import synth, LikelihoodFunction, EngineError
    w = synth.nucleotide_workload(4, 10)
    ambig = np.array([[1.0, 1.0, 0.0, 0.0], [1.0, 0.5, 0.0, 1.0]])
    leaf_states = w.leaf_states.copy()
    leaf_states[0, 0], leaf_states[1, 0] = -1, -2
    with pytest.raises(EngineError, match=r"ambiguity row 1, state 1: weight 0.5 is neither 0 nor 1"):
        LikelihoodFunction(dataclasses.replace(w, ambig=ambig, leaf_states=leaf_states))


def test_product_does_not_import_oracle():
    """The oracle is test infrastructure: nothing under hyphy_b200/ may reference it."""
    for dirpath, _, files in os.walk(os.path.join(ROOT, "hyphy_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                src = open(os.path.join(dirpath, f)).read()
                assert "oracle" not in src.replace("SURVEY", ""), f"{f} mentions the oracle"
