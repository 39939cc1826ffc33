"""CPU emulation of the coset-batched LDE: the first column pass over several cosets of a column group in one launch,
the middle and row passes over all of them, checked bit for bit against the oracle's coset FFT and against the
per-coset path (tests/emu/ntt_cosets_emu.cpp). Catches the indexing of per-coset slabs, tables and pre-weights
without a GPU."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_lde_cosets_batched_on_host(tmp_path):
    import oracle_lib

    oracle_lib.build_oracle()
    exe = str(tmp_path / "gl_ntt_cosets_emu")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-DGL_FORCE_32BIT_PATH", "-o", exe,
                           os.path.join(ROOT, "tests", "emu", "ntt_cosets_emu.cpp"), "-L" + os.path.join(ROOT, "oracle"),
                           "-lgl_oracle", "-Wl,-rpath," + os.path.join(ROOT, "oracle"), "-pthread"])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "COSET EMU OK" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
