"""The restatement of Sage's digest and prefilter (digest_reference) against the CPU oracle (oracle_digest) and against the reference's own
unit tests, without a GPU: every digest_cases case inside Sage's domain, the fast digest_edges cases, the prefilter on small FASTAs, the
26 #[cfg(test)] known answers of enzyme.rs, peptide.rs, modification.rs and database.rs, the FASTA text Rust's str handling decides, and a
sensitivity check that planted mistakes in the restatement are caught."""
import numpy as np
import pytest

import digest_cases as DC
import digest_edges as E
import digest_reference as R
import search_reference as SR
from oracle.oracle import ScorerConfig
from oracle_digest import digest_oracle
from sage_b200 import Peptides, synth

# Cases of digest_cases outside Sage's domain, and why: the reference panics or rejects the file before digesting.
OUTSIDE = {
    "bytes_over_127": R.ReferenceRejects,              # Latin-1 bytes are not UTF-8: read_to_string fails
    "cleave_non_letters": R.ReferencePanics,           # Enzyme::new asserts cleave_at is made of VALID_AA
    "empty_fasta": R.ReferencePanics,                  # group_digests indexes digests[0] of an empty vector
    "header_without_sequence_bare_gt": R.ReferencePanics,   # split_ascii_whitespace().next().unwrap() on a bare '>' with a sequence
    "lowercase_and_odd_letters": R.ReferencePanics,    # skip_suffix[b - b'A'] on the 'w' after a K
}
SLOW_EDGES = {"long_protein_missed3_semi", "accessions_72000"}   # run against the device and the oracle in test_gpu_digest_reference.py


def table_differences(t: dict, o: dict) -> list:
    """The fields where two tables in oracle_digest's layout differ (floats bit for bit, NaN = None)."""
    bad = []
    for k in ("seq_off", "seq", "decoy", "missed", "semi", "prot_off", "name_off"):
        a, b = np.asarray(t[k]).astype(np.int64), np.asarray(o[k]).astype(np.int64)
        if a.shape != b.shape or not np.array_equal(a, b):
            bad.append(k)
    for k in ("mods", "nterm", "cterm", "mono"):
        a, b = DC._bits(np.asarray(t[k], np.float32)), DC._bits(np.asarray(o[k], np.float32))
        if a.shape != b.shape or not np.array_equal(a, b):
            bad.append(k)
    if t["names"][:int(t["name_off"][-1])].tobytes() != o["names"][:int(o["name_off"][-1])].tobytes():
        bad.append("names")
    return bad


def assert_matches_oracle(fasta, kw, what=""):
    t, _ = R.digest_table(fasta, **kw)
    bad = table_differences(t, digest_oracle.digest(fasta, **kw))
    assert not bad, f"{what}: the restatement and the oracle differ in {bad}"
    return t


def test_outside_domain_is_the_documented_list():
    """Every documented case is outside Sage's domain; test_cases_match_oracle fails on any other case that is."""
    for name, exc in OUTSIDE.items():
        fasta, kw = DC.CASES[name]
        with pytest.raises(exc):
            R.digest_table(fasta, **kw)


@pytest.mark.parametrize("name", sorted(DC.CASES))
def test_cases_match_oracle(name):
    if name in OUTSIDE:
        pytest.skip(f"outside Sage's domain: {OUTSIDE[name].__name__}")
    assert_matches_oracle(*DC.CASES[name], what=name)


@pytest.mark.parametrize("name", sorted(set(E.EDGES) - SLOW_EDGES))
def test_edges_match_oracle(name):
    assert_matches_oracle(*E.EDGES[name], what=name)


def test_edge_panics():
    for name, (fasta, kw) in E.EDGE_PANICS.items():
        with pytest.raises(R.ReferencePanics):
            R.digest_table(fasta, **kw)
        t = digest_oracle.digest(fasta, **kw)
        assert len(t["mono"]) == 0, name


# ------------------------------------------------------------------------------------------------ FASTA text as Rust reads it
def test_vertical_tab_is_part_of_the_accession():
    fasta, kw = E.EDGES["vertical_tab_in_header"]
    f = R.fasta_parse(fasta)
    assert [a for a, _ in f.targets] == ["A\x0bB", "A", "C"]   # split_ascii_whitespace does not split at \v; \x0c is ASCII whitespace
    t = assert_matches_oracle(fasta, kw)
    assert any(b"A\x0bB" in x for x in digest_oracle.protein_lists(t))


def test_unicode_whitespace_is_trimmed():
    f = R.fasta_parse(E.EDGES["trailing_nbsp"][0])
    assert [s for _, s in f.targets] == ["PEPTIDEKAAAAAAR", "MWWWWK", "GGGGK"]
    assert R.fasta_parse(E.EDGES["trailing_nbsp_no_newline"][0]).targets == [("A", "PEPTIDEKAAAAAAR")]
    fasta, kw = E.EDGES["trailing_nbsp"]
    t, _ = R.digest_table(fasta, **kw)
    seqs = [t["seq"][t["seq_off"][i]:t["seq_off"][i + 1]].tobytes() for i in range(len(t["mono"]))]
    i = seqs.index(b"AAAAAAR")   # the protein's last peptide: Position Cterm, so the protein C-terminal static mod applies
    assert t["cterm"][i] == np.float32(3.0)
    f = R.fasta_parse(E.EDGES["whitespace_not_trimmed"][0])
    assert [a for a, _ in f.targets] == ["A\x1c", "B\x85C"] and f.targets[0][1].endswith("\x1c")


def test_windows_off_a_character_boundary_are_not_counted():
    fasta, kw = E.EDGES["multibyte_nonspecific"]
    _, st = R.digest_table(fasta, **kw)
    byte_windows = sum(max(len(s.encode()) - L + 1, 0) for _, s in R.fasta_parse(fasta).targets for L in range(5, 8))
    assert st["windows"] < byte_windows
    auto = R.fasta_auto_chunk_size(E.MULTIBYTE, **E.MULTIBYTE_AUTO_KW)
    assert auto == digest_oracle.auto_chunk_size(E.MULTIBYTE, **E.MULTIBYTE_AUTO_KW)
    orig = R.is_char_boundary
    try:
        R.is_char_boundary = lambda raw, i: True   # counting byte windows, as a str::get-less reading would
        assert R.fasta_auto_chunk_size(E.MULTIBYTE, **E.MULTIBYTE_AUTO_KW) != auto
    finally:
        R.is_char_boundary = orig


def test_repeated_variable_spec_keeps_the_last_list():
    P = R.make_parameters(variable_mods={"C": [57.0], "CX": [58.0, 59.0], "M": [15.9949]})
    assert list(P.variable_mods.items()) == [((R.RESIDUE, ord("C")), [np.float32(58.0), np.float32(59.0)]),
                                             ((R.RESIDUE, ord("M")), [np.float32(15.9949)])]


# ------------------------------------------------------------------------------------------------ the prefilter
CFG = dict(precursor_tol=(0, -20.0, 20.0), fragment_tol=(0, -20.0, 20.0))


def _spectra(fasta, kw, n: int, seed: int) -> dict:
    t = digest_oracle.digest(fasta, **kw)
    pep = Peptides(t["seq_off"], t["seq"], t["mods"], t["nterm"], t["mono"], t["decoy"], t["missed"])
    return synth.make_spectra(pep, n, seed=seed, n_peaks=60).as_dict()


def assert_prefilter_matches_oracle(fasta, kw, spectra, chunk, low_memory, cfg=CFG, min_peaks=15):
    t, info = R.prefilter(fasta, spectra, cfg, chunk_size=chunk, low_memory=low_memory, min_peaks=min_peaks, **kw)
    o, oinfo = digest_oracle.prefilter(fasta, spectra, ScorerConfig(**cfg), chunk_size=chunk, low_memory=low_memory, min_peaks=min_peaks, **kw)
    what = f"chunk {chunk} low_memory {low_memory}"
    assert not table_differences(t, o), what
    for k in ("chunk_size", "n_chunks", "plain_build"):
        assert info[k] == oinfo[k], f"{what}: {k}"
    assert np.array_equal(info["rows"], oinfo["rows"]) and np.array_equal(info["kept"], oinfo["kept"]), what
    return t, info


@pytest.mark.parametrize("low_memory", [True, False])
def test_prefilter_matches_oracle(low_memory):
    fasta, kw = E.DECOY_FASTA, E.DECOY_KW
    spectra = _spectra(fasta, kw, 120, 5)
    n = len(R.fasta_parse(fasta).targets)
    for chunk in range(1, n + 1):   # the per-chunk decoy filter at every chunk size
        assert_prefilter_matches_oracle(fasta, kw, spectra, chunk, low_memory)
    fasta, kw = DC.CASES["trypsin_missed1_static_c"]
    spectra = _spectra(fasta, kw, 48, 6)
    for chunk in (3, 7, 39, 0):
        assert_prefilter_matches_oracle(fasta, kw, spectra, chunk, low_memory)


# ------------------------------------------------------------------------------------------------ the reference's known answers
SEQ = "MADEEKLPPGWEKRMSRSSGRVYYFNHITNASQWERPSGN"


def _ep(min_len, max_len, missed, cleave, restrict, c_terminal=True, semi=False):
    return R.EnzymeParameters(missed, min_len, max_len, R.enzyme_new(cleave, restrict, c_terminal, semi))


def _seqs(ep, seq):
    return [d.sequence.decode() for d in R.enzyme_digest(ep, seq, "")]


def _oracle_sequences(seq, min_len, max_len, missed, cleave, restrict, c_terminal=True, semi=False) -> set:
    """The target sequences of the oracle's digest of a one-protein FASTA with the same enzyme (no mass filter, no decoys)."""
    t = digest_oracle.digest(f">A\n{seq}\n", min_len=min_len, max_len=max_len, missed_cleavages=missed, cleave_at=cleave, restrict=restrict,
                             c_terminal=c_terminal, semi_enzymatic=semi, peptide_min_mass=0.0, peptide_max_mass=1e9, generate_decoys=False)
    return {t["seq"][t["seq_off"][i]:t["seq_off"][i + 1]].tobytes().decode() for i in range(len(t["mono"]))}


ENZYME_ANSWERS = {   # enzyme.rs tests: (seq, min_len, max_len, missed, cleave, restrict, c_terminal, semi) -> sequences in order
    "trypsin": ((SEQ, 2, 50, 0, "KR", "P"), ["MADEEK", "LPPGWEK", "MSR", "SSGR", "VYYFNHITNASQWERPSGN"]),
    "trypsin_missed_cleavage": ((SEQ, 0, 50, 1, "KR", "P"), ["MADEEK", "LPPGWEK", "R", "MSR", "SSGR", "VYYFNHITNASQWERPSGN", "MADEEKLPPGWEK",
                                                             "LPPGWEKR", "RMSR", "MSRSSGR", "SSGRVYYFNHITNASQWERPSGN"]),
    "trypsin_missed_cleavage_2": ((SEQ, 0, 50, 2, "KR", "P"), ["MADEEK", "LPPGWEK", "R", "MSR", "SSGR", "VYYFNHITNASQWERPSGN", "MADEEKLPPGWEK",
                                                               "LPPGWEKR", "RMSR", "MSRSSGR", "SSGRVYYFNHITNASQWERPSGN", "MADEEKLPPGWEKR",
                                                               "LPPGWEKRMSR", "RMSRSSGR", "MSRSSGRVYYFNHITNASQWERPSGN"]),
    "test_trypsin_pro": ((SEQ, 2, 50, 0, "KR", ""), ["MADEEK", "LPPGWEK", "MSR", "SSGR", "VYYFNHITNASQWER", "PSGN"]),
    "test_asp_n": ((SEQ + "W", 1, 50, 0, "D", "", False), ["MA", "DEEKLPPGWEKRMSRSSGRVYYFNHITNASQWERPSGNW"]),
    "test_chymotrypsin_pro": ((SEQ + "W", 1, 50, 0, "FYWL", ""), ["MADEEKL", "PPGW", "EKRMSRSSGRVY", "Y", "F", "NHITNASQW", "ERPSGNW"]),
    "no_digest": ((SEQ + "W", 0, 50, 0, "$", ""), [SEQ + "W"]),
    "ensure_unique": (("KVEGAQNQGKKVEGAQNQGK", 2, 50, 0, "KR", ""), ["VEGAQNQGK"]),
    "mini_semi_trypsin": (("MADEEK", 2, 50, 0, "KR", "P", True, True), ["MADEEK", "ADEEK", "MA", "DEEK", "MAD", "EEK", "MADE", "EK", "MADEE"]),
    "semi_trypsin_trypsin_missed_cleavage": (("MADEEKLPPGWEK", 3, 50, 1, "KR", "P", True, True),
                                             ["MADEEK", "LPPGWEK", "MADEEKLPPGWEK", "ADEEK", "DEEK", "MAD", "EEK", "MADE", "MADEE", "PPGWEK", "PGWEK",
                                              "LPP", "GWEK", "LPPG", "WEK", "LPPGW", "LPPGWE", "ADEEKLPPGWEK", "DEEKLPPGWEK", "EEKLPPGWEK",
                                              "EKLPPGWEK", "KLPPGWEK", "MADEEKL", "MADEEKLP", "MADEEKLPP", "MADEEKLPPG", "MADEEKLPPGW",
                                              "MADEEKLPPGWE"]),
}


@pytest.mark.parametrize("name", sorted(ENZYME_ANSWERS))
def test_enzyme_known_answers(name):
    args, expected = ENZYME_ANSWERS[name]
    seq, rest = args[0], args[1:]
    got = _seqs(_ep(*rest), seq)
    assert got == expected
    if name == "no_digest":
        assert _seqs(_ep(0, 10 ** 6, 0, "$", ""), seq) == expected   # max_len usize::MAX in the reference's test
    assert _oracle_sequences(seq, *rest) == set(expected)


def test_enzyme_known_answers_nonspecific():
    s = SEQ + "W"
    assert _seqs(_ep(5, 5, 0, "", ""), s) == [s[i:i + 5] for i in range(len(s) - 4)]
    assert _seqs(_ep(5, 7, 0, "", ""), s) == [s[i:i + L] for L in (5, 6, 7) for i in range(len(s) - L + 1)]   # nonspecific_digest_5_7
    assert _oracle_sequences(s, 5, 7, 0, "", "") == {s[i:i + L] for L in (5, 6, 7) for i in range(len(s) - L + 1)}


def test_enzyme_known_answers_positions_and_missed():
    d = R.enzyme_digest(_ep(2, 50, 0, "KR", "P"), SEQ, "")
    assert [x.position for x in d] == [R.NTERM, R.INTERNAL, R.INTERNAL, R.INTERNAL, R.CTERM]   # trypsin
    # semi_trypsin_trypsin_missed_cleavage and quickcheck_semi_missed_cleavages: missed = interior K/R count
    rng = np.random.default_rng(3)
    for seq in ["MADEEKLPPGWEK"] + ["".join(rng.choice(list(R.VALID_AA.decode()), int(rng.integers(0, 60)))) for _ in range(200)]:
        for x in R.enzyme_digest(_ep(3, 50, 2 if seq != "MADEEKLPPGWEK" else 1, "KR", "" if seq != "MADEEKLPPGWEK" else "P", True, True), seq, ""):
            assert x.missed_cleavages == sum(c in b"KR" for c in x.sequence[::-1][1:]), x.sequence
            if seq == "MADEEKLPPGWEK" and x.sequence.startswith(b"MAD") and x.sequence != seq.encode():
                assert x.position == R.NTERM
    # hash_digest: equality and hashing are (sequence, position)
    assert len({(b"MADEEK", R.NTERM), (b"MADEEK", R.NTERM)}) == 1 and len({(b"MADEEK", R.NTERM), (b"MADEEK", R.INTERNAL)}) == 2


def _pep(seq: str, position=R.INTERNAL):
    return R.peptide_from_digest(R.Digest(False, False, seq.encode(), "", 0, position))


def _var(pep, mods, k, static=()):
    return [p.to_string() for p in R.apply(pep.clone(), [(R.parse_spec(s), np.float32(m)) for s, m in mods], list(static), k)]


def test_peptide_full():
    peps = [R.peptide_from_digest(d) for d in R.enzyme_digest(_ep(0, 50, 0, "KR", "P"), "MPEPTIDEKMSAGEKEND", "")]
    assert [(p.to_string(), p.position) for p in peps] == [("MPEPTIDEK", R.NTERM), ("MSAGEK", R.INTERNAL), ("END", R.CTERM)]
    mods = [("[", 42.0), ("]", 11.0), ("^", 12.0), ("$", 19.0)]
    assert _var(peps[0], mods, 2) == ["MPEPTIDEK", "[+42]-MPEPTIDEK", "[+12]-MPEPTIDEK", "MPEPTIDEK-[+19]", "[+42]-MPEPTIDEK-[+19]",
                                      "[+12]-MPEPTIDEK-[+19]"]
    assert _var(peps[1], mods, 2) == ["MSAGEK", "[+12]-MSAGEK", "MSAGEK-[+19]", "[+12]-MSAGEK-[+19]"]
    assert _var(peps[2], mods, 2) == ["END", "END-[+11]", "[+12]-END", "END-[+19]", "[+12]-END-[+11]", "[+12]-END-[+19]"]


def test_peptide_variable_mods():
    g = _pep("GCMGCMG")
    assert _var(g, [("M", 16.0), ("C", 57.0)], 2) == ["GCMGCMG", "GCM[+16]GCMG", "GCMGCM[+16]G", "GC[+57]MGCMG", "GCMGC[+57]MG",
                                                      "GCM[+16]GCM[+16]G", "GC[+57]M[+16]GCMG", "GCM[+16]GC[+57]MG", "GC[+57]MGCM[+16]G",
                                                      "GCMGC[+57]M[+16]G", "GC[+57]MGC[+57]MG"]
    assert _var(_pep("AAAAAAAA"), [("M", 16.0), ("C", 57.0)], 2) == ["AAAAAAAA"]   # test_variable_mods_no_effeect
    assert _var(g, [("^", 42.0), ("M", 16.0)], 3) == ["GCMGCMG", "[+42]-GCMGCMG", "GCM[+16]GCMG", "GCMGCM[+16]G", "[+42]-GCM[+16]GCMG",
                                                      "[+42]-GCMGCM[+16]G", "GCM[+16]GCM[+16]G", "[+42]-GCM[+16]GCM[+16]G"]
    assert _var(g, [("$", 42.0), ("M", 16.0)], 3) == ["GCMGCMG", "GCMGCMG-[+42]", "GCM[+16]GCMG", "GCMGCM[+16]G", "GCM[+16]GCMG-[+42]",
                                                      "GCMGCM[+16]G-[+42]", "GCM[+16]GCM[+16]G", "GCM[+16]GCM[+16]G-[+42]"]
    assert _var(_pep("GGGSGGGS"), [("S", 79.0), ("S", 541.0)], 2) == ["GGGSGGGS", "GGGS[+79]GGGS", "GGGSGGGS[+79]", "GGGS[+541]GGGS",
                                                                      "GGGSGGGS[+541]", "GGGS[+79]GGGS[+79]", "GGGS[+79]GGGS[+541]",
                                                                      "GGGS[+541]GGGS[+79]", "GGGS[+541]GGGS[+541]"]
    assert _var(_pep("AACAACAA"), [("C", 30.0)], 2, [(R.parse_spec("C"), np.float32(57.0))]) == [   # apply_mods
        "AAC[+57]AAC[+57]AA", "AAC[+30]AAC[+57]AA", "AAC[+57]AAC[+30]AA", "AAC[+30]AAC[+30]AA"]


def test_peptide_modification_sites():
    p = _pep("AACAACAA")
    acc = []
    R.push_resi(p, acc, R.parse_spec("C"), 16.0)
    assert acc == [(2, 16.0), (5, 16.0)]
    for spec, site in (("$", R.SITE_C), ("^", R.SITE_N)):
        acc = []
        R.push_resi(p, acc, R.parse_spec(spec), 16.0)
        assert acc == [(site, 16.0)]
    acc = []
    for spec, mass in (("^", 12.0), ("$", 200.0), ("C", 57.0), ("A", 43.0)):
        R.push_resi(p, acc, R.parse_spec(spec), mass)
    assert acc == [(R.SITE_N, 12.0), (R.SITE_C, 200.0), (2, 57.0), (5, 57.0)] + [(i, 43.0) for i in (0, 1, 3, 4, 6, 7)]


def test_peptide_psuedo_forward():
    for d in R.enzyme_digest(_ep(3, 30, 0, "KR", "P"), SEQ, ""):
        fwd, rev = R.peptide_from_digest(d), R.peptide_from_digest(d.reverse())
        assert not fwd.decoy and rev.decoy
        assert len(fwd.sequence) < 4 or fwd.sequence != rev.sequence
        assert R.reverse(rev).to_string() == fwd.to_string()


def test_modification_parse():
    assert R.parse_spec("[") == (R.PROT_N, -1)
    assert R.parse_spec("[M") == (R.PROT_N, ord("M"))
    assert R.parse_spec("]M") == (R.PROT_C, ord("M"))
    assert R.parse_spec("M") == (R.RESIDUE, ord("M"))
    assert R.parse_spec("Z") is None
    assert R.parse_spec("ABC") is None and R.parse_spec("") is None and R.parse_spec("CX") == (R.RESIDUE, ord("C"))


def test_database_binary_search_slice():
    data = np.array([1.0, 1.5, 2.0, 2.5, 3.0, 3.5, 4.0])
    assert [int(x[0]) for x in SR.binary_search_slice(data, 1.75, 3.5)] == [1, 6]
    assert [int(x[0]) for x in SR.binary_search_slice(data, 0.0, 5.0)] == [0, 7]
    data = np.array([1.0, 1.5, 1.5, 1.5, 1.5, 2.0, 2.5, 3.0, 3.0, 3.5, 4.0])
    lo, hi = (int(x[0]) for x in SR.binary_search_slice(data, 1.5, 3.25))
    assert data[lo] <= 1.5 and data[hi] > 3.25 and list(data[lo:hi]) == [1.0, 1.5, 1.5, 1.5, 1.5, 2.0, 2.5, 3.0, 3.0]


DIGESTION_FASTA = "\n        >sp|AAAAA\n        MEWKLEQSMREQALLKAQLTQLK\n        >sp|BBBBB\n        RMEWKLEQSMREQALLKAQLTQLK\n        "
DIGESTION_KW = dict(missed_cleavages=1, min_len=6, max_len=10, peptide_min_mass=150.0, peptide_max_mass=5000.0, variable_mods={"[": [42.0]},
                    max_variable_mods=2, generate_decoys=False)


def test_database_digestion():
    f = R.fasta_parse(DIGESTION_FASTA, "rev_", False)
    assert f.targets == [("sp|AAAAA", "MEWKLEQSMREQALLKAQLTQLK"), ("sp|BBBBB", "RMEWKLEQSMREQALLKAQLTQLK")]
    for t in (R.digest_table(DIGESTION_FASTA, **DIGESTION_KW)[0], digest_oracle.digest(DIGESTION_FASTA, **DIGESTION_KW)):
        seqs = [t["seq"][t["seq_off"][i]:t["seq_off"][i + 1]].tobytes().decode() for i in range(len(t["mono"]))]
        assert seqs == ["EQALLK", "LEQSMR", "AQLTQLK", "MEWKLEQSMR", "MEWKLEQSMR"]
        assert np.isnan(t["nterm"][:4]).all() and t["nterm"][4] == np.float32(42.0)
        lists = digest_oracle.protein_lists(t)
        assert all(len(x) == 2 for x in lists[:4]) and lists[4] == [b"sp|AAAAA"]


# ------------------------------------------------------------------------------------------------ sensitivity
def _reverse_moves_last(p):
    q = p.clone()
    q.decoy = not p.decoy
    if len(q.sequence) > 2:
        q.sequence = q.sequence[:1] + q.sequence[1:][::-1]
        q.modifications[1:] = q.modifications[1:][::-1]
    return q


MUTATIONS = {   # name -> (attribute of digest_reference, replacement, the case that must then fail)
    "reverse_moves_last_residue": ("reverse", _reverse_moves_last, ("structure", DC.CASES)),
    "mass_filter_exclusive": ("in_mass_range", lambda P, m: bool(m > P.peptide_min_mass and m < P.peptide_max_mass), ("mass_min_at", E.EDGES)),
    "same_site_not_skipped": ("same_site", lambda combination: False, ("two_masses_one_spec", E.EDGES)),
    "ascii_trim": ("rust_trim", lambda s: s.strip(" \t\n\x0b\x0c\r"), ("trailing_nbsp", E.EDGES)),
}


@pytest.mark.parametrize("name", sorted(MUTATIONS))
def test_sensitivity(name, monkeypatch):
    attr, repl, (case, table) = MUTATIONS[name]
    fasta, kw = table[case]
    assert_matches_oracle(fasta, kw, case)
    monkeypatch.setattr(R, attr, repl)
    try:
        t, _ = R.digest_table(fasta, **kw)
    except R.ReferencePanics:
        return   # the case fails: the mutated reading reaches a panic the reference never meets on it
    assert table_differences(t, digest_oracle.digest(fasta, **kw)), f"the mutation {name} went unnoticed on {case}"
