"""The full round's hand-overs between the integer and FP64 pipes, through the host emulation of tests/test_emu.py:
the S-box limbs built as 2^52-offset bit patterns by integer adds (default) or from register-built doubles
(-DGL_SBOX_MOVE_HANDOVER), and the FP64 -> u64 return as a short 2^64 = 2^32 - 1 fold (default) or a 96-bit reduction
(-DGL_RET_REDUCE96). Each form is checked on edge and 2^24 random words against unsigned __int128, and the whole
permutation under each switch against both oracle forms, the reference's known answers and the 2^53 limb bound."""
import pytest

from test_emu import _build_and_run

SWITCHES = [[], ["-DGL_SBOX_MOVE_HANDOVER"], ["-DGL_RET_REDUCE96"], ["-DGL_SBOX_MOVE_HANDOVER", "-DGL_RET_REDUCE96"]]


@pytest.mark.parametrize("defs", SWITCHES, ids=lambda d: "+".join(x[2:] for x in d) or "default")
def test_handover_forms_against_int128(tmp_path, defs):
    out = _build_and_run(tmp_path, "sbox_handover_emu.cpp", "gl_handover_emu", [str(1 << 24)],
                         defs=["-DGL_FP64_ON_HOST", *defs])
    assert "HANDOVER EMU OK" in out, out


@pytest.mark.parametrize("defs", SWITCHES[1:], ids=lambda d: "+".join(x[2:] for x in d))
def test_permutation_under_handover_switch(tmp_path, defs):
    # the default build is test_emu.py's test_poseidon_fp64_pipe_formulation_on_host
    out = _build_and_run(tmp_path, "poseidon_f64_emu.cpp", "gl_f64_emu", ["20000"], defs=["-DGL_FP64_ON_HOST", *defs])
    assert "POSEIDON F64 EMU OK" in out, out
