"""The partial-round pair in both forms through the host emulation of tests/test_emu.py: the renormalisation of the
FP64 limbs on the edges of its input range (tests/emu/poseidon_pair_renorm_emu.cpp), and the former pair
(-DGL_PAIR_RENORM_F64: rank-one terms one by one, renormalisation on the FP64 pipe) through the whole permutation
against both oracle forms. The default pair's permutation is covered by test_emu.py."""
import pytest

from test_emu import _build_and_run


@pytest.mark.parametrize("defs", [[], ["-DGL_PAIR_RENORM_F64"]], ids=["default", "GL_PAIR_RENORM_F64"])
def test_pair_renorm_edges_on_host(tmp_path, defs):
    out = _build_and_run(tmp_path, "poseidon_pair_renorm_emu.cpp", "gl_renorm_emu", ["400000"],
                         defs=["-DGL_FP64_ON_HOST", *defs])
    assert "PAIR RENORM EMU OK" in out, out


def test_poseidon_fp64_with_former_pair(tmp_path):
    out = _build_and_run(tmp_path, "poseidon_f64_emu.cpp", "gl_f64_emu", ["20000"],
                         defs=["-DGL_FP64_ON_HOST", "-DGL_PAIR_RENORM_F64"])
    assert "POSEIDON F64 EMU OK" in out, out
