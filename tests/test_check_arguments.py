"""plonky2's two global arguments checked on a witness: plonk.check_copy_constraints (gl_plonk_check_copies) and
plonk.check_lookups (gl_plonk_check_lookups).

The restatements here follow the reference: copies recover sigma from a dict of identity values k_is[col] * w^row
(permutation_argument.rs:113-157) and compare each routed wire with its sigma's; lookups follow set_lookup_wires
(plonk/prover.rs:50-108), LookupGenerator (gates/lookup.rs:195-220) and LookupTableGenerator
(gates/lookup_table.rs:209-233) line by line.

CPU: the per-thread code of gl_check_args.cuh, run on the host by tests/emu/check_args_emu.cpp, gives the restatements'
failures on the small circuits of tests/plonk_circuits.py (with and without zero knowledge, with lookups, with copies
through virtual targets), honest and broken; the Python entry points refuse bad shapes before any device work.

GPU (-m gpu): honest witnesses give no failure; copy and lookup violations give exactly the expected entries; every
report equals the restatement's, truncation included; the checks agree with check_constraints under the proof's
challenges; non-canonical, page-locked and still-in-production witnesses; sigmas that are not a permutation."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import gl_numpy as gn
import plonk_circuits as PC
from test_circuit_data import sigma_values, vector_sigma_map

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = PC.P


def _plonk():
    from plonky2_b200 import plonk

    return plonk


# ------------------------------------------------------------------------------------------------ restatements
def restated_copies(wires, sigmas, k_is, degree_bits):
    """Every failing (i, sigma(i)), i = row * num_routed + col ascending: sigma from a dict of identity values."""
    nr, n = sigmas.shape
    subgroup = gn.powers(PC.root_of_unity(degree_bits), n)
    where = {}
    for col in range(nr):
        for row, v in enumerate(gn.mul(np.full(n, k_is[col], dtype=np.uint64), subgroup).tolist()):
            where[v] = row * nr + col
    out = []
    for row in range(n):
        for col in range(nr):
            j = where[int(sigmas[col, row]) % P]
            if int(wires[col, row]) % P != int(wires[j % nr, j // nr]) % P:
                out.append((row * nr + col, j))
    return out


def restated_lookups(cd, wires):
    """Every lookup failure as (row, 4 * slot + kind) in order, and every entry's count (a list per table)."""
    nr = cd.config.num_routed_wires
    num_entries, num_lut_entries = nr // 2, nr // 3               # LookupGate / LookupTableGate::num_slots
    w = lambda c, r: int(wires[c, r]) % P                        # noqa: E731
    fails, all_counts = [], []
    for lut, (last_lu, last_lut, first_lut) in zip(cd.luts, cd.lookup_rows):
        lut = [tuple(e) for e in lut]
        table_value_to_idx = {inp: i for i, (inp, _) in enumerate(lut)}   # a later entry of one input wins
        multiplicities = [0] * len(lut)
        # the padding of the last LookupGate with the first entry: the run of slots at the end of row last_lut - 1
        pad_from = num_entries
        while pad_from > 0 and (w(2 * (pad_from - 1), last_lut - 1), w(2 * pad_from - 1, last_lut - 1)) == lut[0]:
            pad_from -= 1
        for row in range(last_lu, last_lut):
            for slot in range(num_entries):
                pair = (w(2 * slot, row), w(2 * slot + 1, row))
                if row == last_lut - 1 and slot >= pad_from:
                    multiplicities[0] += 1
                elif pair[0] in table_value_to_idx:
                    multiplicities[table_value_to_idx[pair[0]]] += 1
                if pair not in lut:                                       # "Incorrect input value provided"
                    fails.append((row, 4 * slot + 1))
        for row in range(last_lut, first_lut + 1):
            for slot in range(num_lut_entries):
                e = (first_lut - row) * num_lut_entries + slot
                want = lut[e] if e < len(lut) else lut[0]
                if (w(3 * slot, row), w(3 * slot + 1, row)) != want:
                    fails.append((row, 4 * slot + 2))
                if w(3 * slot + 2, row) != (multiplicities[e] if e < len(lut) else 0):
                    fails.append((row, 4 * slot + 3))
        all_counts.append(multiplicities)
    return sorted(fails), all_counts


# ------------------------------------------------------------------------------------------------ circuits
def circuits():
    """(name, circuit) of the small test circuits: every shape, zero knowledge with and without lookups."""
    plonk = _plonk()
    out = [("shape%d" % k, PC.shape_circuit(s, 2)) for k, s in enumerate(PC.SHAPES)]
    out.append(("lookup64", PC.shape_circuit(PC.LOOKUP_64, 2)))
    zk = plonk.standard_recursion_zk_config()
    for lookups in (False, True):
        c, _ = PC.zk_circuit(plonk, zk, PC.quick_fri_config(zk), lookups=lookups)
        out.append(("zk" + ("_lookups" if lookups else ""), c))
    return out


def with_virtual_cycle(c, wires_list):
    """c with one more copy set: the (row, col) wires of wires_list, joined only through one virtual target, all
    carrying the value of the first. Returns the new sigmas (c.wires is updated)."""
    cd, cfg = c.common, c.config
    nw, n = cfg.num_wires, c.n
    v = n * nw                                                     # virtual target 0
    pairs = np.concatenate([PC.pairs_from_sigmas(c), [[r * nw + col, v] for r, col in wires_list]])
    for r, col in wires_list[1:]:
        c.wires[col, r] = c.wires[wires_list[0][1], wires_list[0][0]]
    return sigma_values(vector_sigma_map(nw, cfg.num_routed_wires, cd.degree_bits, 1, pairs), cd.k_is, cd.degree_bits)


def lookup_mutations(c):
    """(name, wires, the expected (row, 4 * slot + kind)) of the four lookup violations, on table 0 of c."""
    cd = c.common
    nr = cd.config.num_routed_wires
    nts = nr // 3
    lut = cd.luts[0]
    last_lu, last_lut, first_lut = cd.lookup_rows[0]
    where = lambda e: (first_lut - e // nts, e % nts)                # noqa: E731
    idx = {inp: i for i, (inp, _) in enumerate(lut)}
    out = []
    w = c.wires.copy()                                               # a multiplicity off by one
    r, s = where(3)
    w[3 * s + 2, r] = (int(w[3 * s + 2, r]) + 1) % P
    out.append(("multiplicity", w, [(r, 4 * s + 3)]))
    w = c.wires.copy()                                               # a changed table slot (its entry's input + 1)
    r, s = where(5)
    w[3 * s, r] = (int(w[3 * s, r]) + 1) % P
    out.append(("table", w, [(r, 4 * s + 2)]))
    w = c.wires.copy()                                               # a looked input with the wrong output
    row, slot = last_lu, 1
    w[2 * slot + 1, row] = (int(w[2 * slot + 1, row]) + 1) & 0xFFFF
    out.append(("output", w, [(row, 4 * slot + 1)]))
    w = c.wires.copy()                                               # a looked pair moved outside the table
    e = idx[int(w[2 * slot, row])]
    w[2 * slot, row] = 0                                             # inputs are 3e + 1 or 7e + 2: never 0
    r, s = where(e)
    out.append(("moved", w, sorted([(row, 4 * slot + 1), (r, 4 * s + 3)])))
    return out


# ------------------------------------------------------------------------------------------------------ CPU
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("gl_check_args_emu") / "libgl_check_args_emu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-DGL_FORCE_32BIT_PATH", "-shared", "-fPIC", "-o", out,
                           os.path.join(ROOT, "tests", "emu", "check_args_emu.cpp")])
    L = C.CDLL(out)
    L.emu_check_copies.restype = C.c_uint64
    L.emu_check_lookups.restype = C.c_uint64
    return L


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def emu_copies(L, wires, sigmas, k_is, degree_bits):
    nr, n = sigmas.shape
    w = np.ascontiguousarray(wires[:nr], dtype=np.uint64)
    s = np.ascontiguousarray(sigmas, dtype=np.uint64)
    k = np.array(k_is, dtype=np.uint64)
    pairs = np.zeros(2 * nr * n, dtype=np.uint32)
    total = L.emu_check_copies(_ptr(w), _ptr(s), _ptr(k), degree_bits, nr, _ptr(pairs))
    assert total != 2**64 - 1, "not a permutation"
    return [(int(a), int(b)) for a, b in pairs[:2 * total].reshape(-1, 2)]


def emu_lookups(L, cd, wires):
    nr, n = cd.config.num_routed_wires, 1 << cd.degree_bits
    w = np.ascontiguousarray(wires, dtype=np.uint64)
    luts = np.ascontiguousarray(np.concatenate([np.array(t, dtype=np.uint16) for t in cd.luts]), dtype=np.uint16)
    offsets = np.concatenate([[0], np.cumsum([len(t) for t in cd.luts])]).astype(np.uint32)
    rows = np.array(cd.lookup_rows, dtype=np.uint32).reshape(-1)
    counts = np.zeros(int(offsets[-1]), dtype=np.uint32)
    pairs = np.zeros(2 * nr * n, dtype=np.uint32)
    total = L.emu_check_lookups(_ptr(w), cd.degree_bits, nr, _ptr(luts), _ptr(offsets), _ptr(rows), len(cd.luts),
                                _ptr(counts), _ptr(pairs))
    got = [(int(a), int(b)) for a, b in pairs[:2 * total].reshape(-1, 2)]
    return got, [counts[offsets[k]:offsets[k + 1]].tolist() for k in range(len(cd.luts))]


def _break_wires(c, rng, count):
    w = c.wires.copy()
    nr = c.config.num_routed_wires
    for _ in range(count):
        col, row = int(rng.integers(0, nr)), int(rng.integers(0, c.n))
        w[col, row] = (int(w[col, row]) + 1 + int(rng.integers(0, 3))) % P
    return w


@pytest.mark.parametrize("name,c", circuits(), ids=lambda v: v if isinstance(v, str) else "")
def test_copies_on_host_are_the_restatement(emu, name, c):
    """Honest: no failure. Then random wires changed: the host run of the kernels' code gives the restatement's pairs."""
    cd = c.common
    assert emu_copies(emu, c.wires, c.sigmas, cd.k_is, cd.degree_bits) == []
    rng = np.random.default_rng(len(name))
    w = _break_wires(c, rng, 6)
    want = restated_copies(w, c.sigmas, cd.k_is, cd.degree_bits)
    assert emu_copies(emu, w, c.sigmas, cd.k_is, cd.degree_bits) == want
    nonc = np.where(w < np.uint64(2**32 - 1), w + np.uint64(P), w)    # non-canonical witness, same residues
    assert emu_copies(emu, nonc, c.sigmas, cd.k_is, cd.degree_bits) == want


def test_copies_through_a_virtual_target_on_host(emu):
    """A set joined only through a virtual target, across the first and last rows and the last routed column."""
    c = PC.shape_circuit(PC.RECURSION_5, 2)
    cd, nr, n = c.common, c.config.num_routed_wires, c.n
    sig = with_virtual_cycle(c, [(0, nr - 1), (n - 1, 5), (n - 2, nr - 1)])
    assert emu_copies(emu, c.wires, sig, cd.k_is, cd.degree_bits) == []
    assert restated_copies(c.wires, sig, cd.k_is, cd.degree_bits) == []
    w = c.wires.copy()
    w[nr - 1, 0] = (int(w[nr - 1, 0]) + 1) % P
    got = emu_copies(emu, w, sig, cd.k_is, cd.degree_bits)
    assert got == restated_copies(w, sig, cd.k_is, cd.degree_bits)
    i = nr - 1                                                       # wire (0, nr - 1)
    assert len(got) == 2 and got[0][0] == i and got[1][1] == i


@pytest.mark.parametrize("name", ["shape6", "lookup64", "zk_lookups"])
def test_lookups_on_host_are_the_restatement(emu, name):
    """Honest: no failure and the recorded multiplicities are the counts. Each violation: the expected entries, equal
    to the restatement's."""
    c = dict(circuits())[name]
    cd = c.common
    got, counts = emu_lookups(emu, cd, c.wires)
    want, want_counts = restated_lookups(cd, c.wires)
    assert got == want == [] and counts == want_counts
    for what, w, expected in lookup_mutations(c):
        got, counts = emu_lookups(emu, cd, w)
        want, want_counts = restated_lookups(cd, w)
        assert got == want == expected, what
        assert counts == want_counts, what


def test_restated_padding_counts_for_entry_zero(emu):
    """A LUT whose first input repeats later: the padding run of the last LookupGate row counts for entry 0, a looked
    input for its later entry (both the host run and the restatement)."""
    c = PC.shape_circuit(PC.LOOKUP_64, 2)
    cd = c.common
    lut = [tuple(e) for e in cd.luts[0]]
    lut[7] = (lut[0][0], lut[7][1])                                  # entry 7 shares entry 0's input
    cd.luts[0] = lut
    got, counts = emu_lookups(emu, cd, c.wires)
    want, want_counts = restated_lookups(cd, c.wires)
    assert got == want and counts == want_counts


# lookup configs whose witness has fewer than 1.5 x num_routed_wires columns: looking slot s has no column 3s + 2
NARROW = [(80, 80, 8, 3, 5, 0, (), True), (100, 80, 8, 3, 5, 0, (), True)]


def last_slot_mutations(c):
    """(name, wires, the expected (row, 4 * slot + kind)) of L1 failures in the last looking slot of the first
    LookupGate row: a wrong output, and an input moved outside the table (with the L3 of the entry it counted for)."""
    cd = c.common
    nts, slot = cd.config.num_routed_wires // 3, cd.config.num_routed_wires // 2 - 1
    last_lu, _, first_lut = cd.lookup_rows[0]
    idx = {inp: i for i, (inp, _) in enumerate(cd.luts[0])}
    w = c.wires.copy()
    w[2 * slot + 1, last_lu] = (int(w[2 * slot + 1, last_lu]) + 1) & 0xFFFF
    out = [("output", w, [(last_lu, 4 * slot + 1)])]
    w = c.wires.copy()
    e = idx[int(w[2 * slot, last_lu])]
    w[2 * slot, last_lu] = 0                                         # inputs are 3e + 1: never 0
    out.append(("moved", w, sorted([(last_lu, 4 * slot + 1), (first_lut - e // nts, 4 * (e % nts) + 3)])))
    return out


class _HostOnlyCtx:
    """A context stand-in for check_lookups on a host witness whose native call is replaced."""
    h = None


@pytest.mark.parametrize("shape", NARROW, ids=["80-80", "100-80"])
def test_narrow_witness_with_l1_in_the_last_looking_slot(emu, monkeypatch, shape):
    """A lookup config with num_wires < 1.5 x num_routed_wires (e.g. CircuitConfig(num_wires=80, num_routed_wires=80)),
    an L1 failure in the last looking slot: the host run gives the restatement's entries, and check_lookups labels
    them from the host witness without reading a multiplicity column the looking slot does not have (the native call
    is replaced by the host run here, so that the labelling runs without a device)."""
    from plonky2_b200 import _native as N

    plonk = _plonk()
    c = PC.shape_circuit(shape, 2)
    cd, nr = c.common, c.config.num_routed_wires
    assert 3 * (nr // 2 - 1) + 2 >= c.wires.shape[0]
    for what, w, expected in last_slot_mutations(c):
        got, counts = emu_lookups(emu, cd, w)
        assert got == expected == restated_lookups(cd, w)[0], what

        class HostRun:
            @staticmethod
            def gl_plonk_check_lookups(*a):
                counts_out, max_report, failures, pairs_out, reported = a[10], a[11], a[12], a[13], a[14]
                flat = [v for t in counts for v in t]
                for i, v in enumerate(flat):
                    counts_out[i] = v
                failures._obj.value = len(got)
                reported._obj.value = min(len(got), max_report)
                for i, (r, code) in enumerate(got[:max_report]):
                    pairs_out[2 * i], pairs_out[2 * i + 1] = r, code
                return N.GL_OK
        monkeypatch.setattr(N, "lib", lambda: HostRun)
        rep = plonk.check_lookups(cd, w, ctx=_HostOnlyCtx)
        monkeypatch.undo()
        assert _lookup_pairs(rep) == expected, what
        row, slot, label = rep.entries[[k for _, k in expected].index(4 * (nr // 2 - 1) + 1)]
        pair = (int(w[2 * slot, row]), int(w[2 * slot + 1, row]))
        want = "lookup table 0, L1: looking slot (%d, %d) holds (%d, %d), which is not an entry of the table"
        assert label == want % (row, slot, *pair), what


def test_refusals_before_device_work(monkeypatch):
    """Wrong witness or sigmas shapes and max_report outside 0..65536 are ShapeErrors raised before any context is
    created."""
    from plonky2_b200 import _native as N

    plonk = _plonk()

    def no_device(*a, **k):
        raise AssertionError("device work before the refusal")
    monkeypatch.setattr(N, "default_context", no_device)
    c = PC.shape_circuit(PC.LOOKUP_64, 2)
    cd = c.common

    class Data:
        sigmas = c.sigmas
    for bad in (c.wires[:-1], c.wires[:, :-1], c.wires[:, :, None]):
        with pytest.raises(N.ShapeError):
            plonk.check_copy_constraints(Data, cd, bad)
        with pytest.raises(N.ShapeError):
            plonk.check_lookups(cd, bad)
    Data.sigmas = c.sigmas[:-1]
    with pytest.raises(N.ShapeError, match="sigmas"):
        plonk.check_copy_constraints(Data, cd, c.wires)
    Data.sigmas = c.sigmas
    for bad in (-1, N.MAX_REPORT + 1, 1.5):
        with pytest.raises(N.ShapeError, match="max_report"):
            plonk.check_copy_constraints(Data, cd, c.wires, max_report=bad)
        with pytest.raises(N.ShapeError, match="max_report"):
            plonk.check_lookups(cd, c.wires, max_report=bad)


# ------------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def pb():
    import torch

    if not torch.cuda.is_available():
        if os.environ.get("GL_REQUIRE_GPU") == "1":
            raise AssertionError("GPU tests need a CUDA device")
        pytest.skip("no CUDA device (gpu-marked tests run on an H100)")
    import plonky2_b200 as p

    p.default_context()
    return p


class _Data:
    def __init__(self, sigmas):
        self.sigmas = sigmas


def _copy_pairs(report, nr):
    return [(r * nr + col, int(lbl.split(" is copied to wire (")[1].split(",")[0]) * nr
             + int(lbl.split(" is copied to wire (")[1].split(",")[1].split(")")[0])) for r, col, lbl in report.entries]


def _lookup_pairs(report):
    kinds = {"L1": 1, "L2": 2, "L3": 3}
    return [(r, 4 * s + kinds[lbl.split(", ")[1][:2]]) for r, s, lbl in report.entries]


@pytest.mark.gpu
def test_honest_witnesses_have_no_failure(pb):
    plonk = _plonk()
    for name, c in circuits():
        rc = plonk.check_copy_constraints(_Data(c.sigmas), c.common, c.wires)
        assert rc.failures == 0 and rc.entries == [] and rc, name
        if c.common.luts:
            rl = plonk.check_lookups(c.common, c.wires)
            assert rl.failures == 0 and rl, name


@pytest.mark.gpu
def test_large_circuit_2_18_has_no_failure(pb):
    import plonk_large as PL

    plonk = _plonk()
    c = PL.large_circuit(18, luts="range16")
    assert plonk.check_copy_constraints(_Data(c.sigmas), c.common, c.wires).failures == 0
    assert plonk.check_lookups(c.common, c.wires).failures == 0
    w = c.wires.copy()                                               # one copied wire changed: two edges
    R, C_ = c.cycles[0]
    r, col = int(R[1, 0]), int(C_[1, 0])
    w[col, r] = (int(w[col, r]) + 1) % P
    rep = plonk.check_copy_constraints(_Data(c.sigmas), c.common, w)
    nr = c.config.num_routed_wires
    i = r * nr + col
    assert rep.failures == 2 and sorted(p for e in _copy_pairs(rep, nr) for p in e).count(i) == 2


@pytest.mark.gpu
def test_copy_violations(pb):
    """A cycle of length >= 3, a 2-cycle of zero knowledge's Z pairs, a set joined only through a virtual target across
    the first and last rows and the last routed column: one changed wire gives exactly its two edges."""
    plonk = _plonk()
    c = PC.shape_circuit(PC.RECURSION_5, 2)
    nr, n = c.config.num_routed_wires, c.n
    cases = []
    w = c.wires.copy()                                               # the set of the constant 1: long cycle
    w[1, 3] = (int(w[1, 3]) + 5) % P
    cases.append((c.sigmas, w, 3 * nr + 1))
    sig = with_virtual_cycle(c, [(0, nr - 1), (n - 1, 5), (n - 2, nr - 1)])
    for r, col in [(0, nr - 1), (n - 1, 5), (n - 2, nr - 1)]:
        w = c.wires.copy()
        w[col, r] = (int(w[col, r]) + 1) % P
        cases.append((sig, w, r * nr + col))
    c2 = PC.shape_circuit(PC.RECURSION_5, 2)
    sig2 = with_virtual_cycle(c2, [(n - 1, 0), (n - 3, nr - 1)])    # a pair joined only through the virtual target
    w = c2.wires.copy()
    w[0, n - 1] = (int(w[0, n - 1]) + 1) % P
    cases.append((sig2, w, (n - 1) * nr))
    zk = plonk.standard_recursion_zk_config()
    cz, (regular, z_pairs) = PC.zk_circuit(plonk, zk, PC.quick_fri_config(zk))
    r1 = 2 + 12 + regular                                            # the first Z pair
    w = cz.wires.copy()
    w[7, r1] = (int(w[7, r1]) + 1) % P
    cases.append((cz.sigmas, w, r1 * nr + 7, cz))
    for case in cases:
        sigmas, w, i = case[:3]
        circ = case[3] if len(case) > 3 else c
        rep = plonk.check_copy_constraints(_Data(sigmas), circ.common, w)
        got = _copy_pairs(rep, nr)
        assert got == restated_copies(w, sigmas, circ.common.k_is, circ.common.degree_bits)
        assert rep.failures == 2 and [a for a, _ in got].count(i) == 1 and [b for _, b in got].count(i) == 1
        a, b = got[0] if got[0][0] == i else got[1]
        assert rep.entries[[x for x, _ in got].index(i)][2] == "wire (%d, %d) = %d is copied to wire (%d, %d) = %d" % (
            i // nr, i % nr, int(w[i % nr, i // nr]) % P, b // nr, b % nr, int(w[b % nr, b // nr]) % P)


@pytest.mark.gpu
def test_lookup_violations(pb):
    plonk = _plonk()
    for name in ("lookup64", "zk_lookups"):
        c = dict(circuits())[name]
        for what, w, expected in lookup_mutations(c):
            rep = plonk.check_lookups(c.common, w)
            assert rep.failures == len(expected), (name, what)
            assert _lookup_pairs(rep) == expected == restated_lookups(c.common, w)[0], (name, what)
            assert all(lbl.startswith("lookup table 0, L") for _, _, lbl in rep.entries)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", NARROW, ids=["80-80", "100-80"])
def test_narrow_witness_with_l1_in_the_last_looking_slot_on_device(pb, shape):
    """num_wires < 1.5 x num_routed_wires with an L1 failure in the last looking slot, from a host witness and from a
    CUDA tensor: exactly the expected entries, labelled with the looking slot's pair."""
    from test_gpu_stream_order import _dev

    plonk = _plonk()
    c = PC.shape_circuit(shape, 2)
    cd, nr = c.common, c.config.num_routed_wires
    assert plonk.check_lookups(cd, c.wires).failures == 0
    for what, w, expected in last_slot_mutations(c):
        for witness in (w, _dev(w)):
            rep = plonk.check_lookups(cd, witness)
            assert rep.failures == len(expected) and _lookup_pairs(rep) == expected, what
            row, slot, label = rep.entries[[k for _, k in expected].index(4 * (nr // 2 - 1) + 1)]
            assert "holds (%d, %d), which is not" % (int(w[2 * slot, row]), int(w[2 * slot + 1, row])) in label


@pytest.mark.gpu
@pytest.mark.parametrize("max_report", [0, 1, 64, 65536])
def test_reports_equal_the_restatement_with_truncation(pb, max_report):
    plonk = _plonk()
    rng = np.random.default_rng(max_report)
    c = PC.shape_circuit(PC.LOOKUP_64, 2)
    cd, nr = c.common, c.config.num_routed_wires
    w = _break_wires(c, rng, 200)
    want = restated_copies(w, c.sigmas, cd.k_is, cd.degree_bits)
    rep = plonk.check_copy_constraints(_Data(c.sigmas), cd, w, max_report=max_report)
    assert rep.failures == len(want) and _copy_pairs(rep, nr) == want[:max_report]
    want, _ = restated_lookups(cd, w)
    rep = plonk.check_lookups(cd, w, max_report=max_report)
    assert rep.failures == len(want) > 1 and _lookup_pairs(rep) == want[:max_report]


@pytest.mark.gpu
def test_agreement_with_check_constraints(pb):
    """Under the proof's own challenges: copy failures iff check_constraints reports the permutation's closing term,
    lookup failures iff it reports a lookup term."""
    from plonky2_b200 import _native as N

    plonk = _plonk()
    cfg = plonk.CircuitConfig(num_wires=135, num_routed_wires=80, cap_height=3)
    variants = [{}, dict(break_copy=True), dict(break_lookup="pair"), dict(break_lookup="table"), dict(break_gate=True)]
    for kw in variants:
        c = PC.FibonacciCircuit(plonk, cfg, 6, poseidon_rows=4, public_inputs=[3, 1, 4, 1, 5], lookups=True, **kw)
        data = plonk.build_circuit_data(cfg, PC.quick_fri_config(cfg), PC.instances_of(c), PC.pairs_from_sigmas(c),
                                        luts=c.common.luts, lookup_rows=c.lookup_rows)
        try:
            copies = plonk.check_copy_constraints(data.prover_only, data.common, c.wires)
            lookups = plonk.check_lookups(data.common, c.wires)
            labels = []
            try:
                plonk.prove_with_witness(data.prover_only, data.common, c.wires, c.public_inputs,
                                         check_constraints=True)
            except N.ConstraintError as e:
                labels = [lbl for _, _, lbl in e.report.entries]
            assert bool(copies.failures) == any("the permutation does not close" in lbl for lbl in labels), kw
            assert bool(lookups.failures) == any(lbl.startswith("lookup term") for lbl in labels), kw
        finally:
            data.prover_only.constants_sigmas_commitment.close()


@pytest.mark.gpu
def test_input_contracts(pb):
    """Non-canonical witnesses give the canonical witness's report; a page-locked witness and sigmas overwritten as
    soon as the call returns were read before; a CUDA witness still in production is read after its producer."""
    import torch
    from test_gpu_host_buffers import _hold, _host_buffer, _noncanonical, _overwrite
    from test_gpu_stream_order import _delayed, _dev

    plonk = _plonk()
    c = PC.shape_circuit(PC.LOOKUP_64, 2)
    cd = c.common
    w = _break_wires(c, np.random.default_rng(3), 30)
    want_c = plonk.check_copy_constraints(_Data(c.sigmas), cd, w, max_report=1000)
    want_l = plonk.check_lookups(cd, w, max_report=1000)
    assert want_c.failures and want_l.failures
    nonc = _noncanonical(w)
    assert repr(plonk.check_copy_constraints(_Data(_noncanonical(c.sigmas)), cd, nonc, max_report=1000)) == repr(want_c)
    assert repr(plonk.check_lookups(cd, nonc, max_report=1000)) == repr(want_l)
    ctx = pb.default_context()
    for host in ("pinned", "pageable"):
        hw, hs = _host_buffer(w, host), _host_buffer(c.sigmas, host)
        _hold(ctx)
        got = plonk.check_copy_constraints(_Data(hs), cd, hw, max_report=1000)
        _overwrite(hw, hs)
        assert got.failures == want_c.failures
        hw = _host_buffer(w, host)
        _hold(ctx)
        got_l = plonk.check_lookups(cd, hw, max_report=0)
        _overwrite(hw)
        assert got_l.failures == want_l.failures
    # a CUDA witness still in production: the destination first holds the honest witness
    dst, src = _dev(c.wires), _dev(w)
    _delayed((dst, src))
    got = plonk.check_copy_constraints(_Data(c.sigmas), cd, dst, max_report=1000)
    assert repr(got) == repr(want_c)
    dst = _dev(c.wires)
    _delayed((dst, src))
    assert repr(plonk.check_lookups(cd, dst, max_report=1000)) == repr(want_l)
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_corrupt_sigmas_are_refused(pb):
    """Sigmas that are not a permutation of the identity values: GL_ERR_BAD_ARG."""
    from plonky2_b200 import _native as N

    plonk = _plonk()
    c = PC.shape_circuit(PC.RECURSION_5, 2)
    cd, nr = c.common, c.config.num_routed_wires
    for corrupt in ("duplicate", "foreign"):
        s = c.sigmas.copy()
        s[3, 5] = s[4, 6] if corrupt == "duplicate" else 12345
        with pytest.raises(N.NativeError, match="not a permutation"):
            plonk.check_copy_constraints(_Data(s), cd, c.wires)
        ctx = pb.default_context()
        w, k = np.ascontiguousarray(c.wires), np.array(cd.k_is, dtype=np.uint64)
        f, r = C.c_uint64(), C.c_uint32()
        rc = N.lib().gl_plonk_check_copies(ctx.h, N.np_ptr(w), c.n, N.MEM_HOST, N.np_ptr(s), c.n, N.MEM_HOST,
                                           N.np_ptr(k), cd.degree_bits, nr, 0, C.byref(f), None, C.byref(r))
        assert rc == N.GL_ERR_BAD_ARG
