"""The S-box's FP64 hand-over in its former form (-DGL_SBOX_I2F: the four product words through u32 -> double
conversions instead of 2^52-offset doubles) through the same host emulation as tests/test_emu.py, against both oracle
forms. The default form is covered by test_emu.py's test_poseidon_fp64_pipe_formulation_on_host. The squaring switch
(GL_SBOX_SQR4) has no host counterpart: with -DGL_FORCE_32BIT_PATH both squarings are the same three-product C
restatement, and the device asm of sqr_wide_3w runs only on the GPU (the Poseidon KATs of test_gpu_parity.py)."""
from test_emu import _build_and_run


def test_poseidon_fp64_with_i2f_sbox_handover(tmp_path):
    out = _build_and_run(tmp_path, "poseidon_f64_emu.cpp", "gl_f64_emu", ["20000"],
                         defs=["-DGL_FP64_ON_HOST", "-DGL_SBOX_I2F"])
    assert "POSEIDON F64 EMU OK" in out, out
