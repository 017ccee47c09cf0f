"""The oracle's prefilter (oracle_digest.prefilter, auto_chunk_size) on its own: a chunk size covering every protein is the plain digest,
the low_memory=False keep set contains the low_memory=True one, and the automatic chunk size equals a hand computation."""
import numpy as np

import digest_cases as DC
from oracle.oracle import ScorerConfig
from oracle_digest import digest_oracle
from sage_b200 import Peptides, synth

FASTA = DC.random_fasta(30, 31)
KW = dict(missed_cleavages=1, static_mods={"C": 57.021464}, variable_mods={"M": [15.9949]})
CFG = ScorerConfig(precursor_tol=(0, -20.0, 20.0), fragment_tol=(0, -20.0, 20.0))


def _spectra(t: dict, n: int, seed: int) -> dict:
    pep = Peptides(t["seq_off"], t["seq"], t["mods"], t["nterm"], t["mono"], t["decoy"], t["missed"])
    return synth.make_spectra(pep, n, seed=seed, n_peaks=60).as_dict()


def _rows(t: dict) -> set:
    raw = t["seq"].tobytes()
    so = t["seq_off"]
    return {(raw[so[i]:so[i + 1]], t["mods"][so[i]:so[i + 1]].tobytes(), t["nterm"][i].tobytes(), t["cterm"][i].tobytes()) for i in range(len(so) - 1)}


def test_chunk_size_covering_every_protein_is_the_plain_digest():
    plain = digest_oracle.digest(FASTA, **KW)
    spectra = _spectra(plain, 64, 5)
    for cs in (30, 31, 1000):
        t, info = digest_oracle.prefilter(FASTA, spectra, CFG, chunk_size=cs, **KW)
        assert info["plain_build"] == 1 and info["n_chunks"] == 0 and info["chunk_size"] == cs
        for k in plain:
            assert np.array_equal(np.asarray(plain[k]).view(np.uint8), np.asarray(t[k]).view(np.uint8)), k


def test_full_keep_set_contains_low_memory_keep_set():
    plain = digest_oracle.digest(FASTA, **KW)
    spectra = _spectra(plain, 200, 6)
    for cs in (1, 4, 7):
        lo, ilo = digest_oracle.prefilter(FASTA, spectra, CFG, chunk_size=cs, low_memory=True, **KW)
        hi, ihi = digest_oracle.prefilter(FASTA, spectra, CFG, chunk_size=cs, low_memory=False, **KW)
        assert ilo["n_chunks"] == ihi["n_chunks"] == (30 + cs - 1) // cs
        assert np.array_equal(ilo["rows"], ihi["rows"])
        assert (ilo["kept"] <= ihi["kept"]).all() and ilo["kept"].sum() > 0
        assert _rows(lo) <= _rows(hi)


def test_auto_chunk_size_by_hand():
    # two proteins, no enzyme, lengths 7..12: every distinct window of each protein is one unmodified peptide of fasta.digest()
    rng = np.random.default_rng(9)
    a, b = ("".join(rng.choice(list(DC.AA), 800)) for _ in range(2))
    fasta = f">A\n{a}\n>B\n{b}\n>C\n{a}\n"
    kw = dict(cleave_at="", min_len=7, max_len=12, variable_mods={"M": [15.9949, 31.98], "S": [79.966331], "T": [79.966331], "Y": [79.966331],
                                                                  "^": [42.0], "C": [1.0], "W": [3.0], "K": [8.0], "R": [10.0]}, max_variable_mods=8)
    total = sum(len({s[i:i + L] for L in range(7, 13) for i in range(len(s) - L + 1)}) for s in (a, b, a))
    specs = 9   # "M" with two masses is one spec
    count = (specs + 1) * (1 << 8) * total // (1 << 23)
    assert count >= 1
    expect = 3 // count if count else 3
    assert digest_oracle.auto_chunk_size(fasta, **kw) == expect
    kw2 = dict(kw, max_variable_mods=2)
    assert digest_oracle.auto_chunk_size(fasta, **kw2) == 3   # (10 * 4 * total) // 2^23 == 0: the whole FASTA is one chunk
