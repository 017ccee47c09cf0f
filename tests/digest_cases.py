"""Workloads of the device digest (sage_b200.digest_fasta): each case is FASTA text (str or bytes) and the digest keywords, checked against
the CPU oracle's digest() (oracle_digest). Names say what each case pins."""
from __future__ import annotations

import numpy as np

AA = "ACDEFGHIKLMNPQRSTVWY"
# SwissProt residue frequencies (%), in AA order
FREQ = np.array([8.25, 1.37, 5.45, 6.75, 3.86, 7.07, 2.27, 5.96, 5.84, 9.66, 2.42, 4.06, 4.70, 3.93, 5.53, 6.56, 5.34, 6.87, 1.08, 2.92])


def random_fasta(n: int, seed: int, median: float = 375.0, lo: int = 30, hi: int = 5000, prefix: str = "sp|P") -> str:
    """n seeded proteins with lognormal lengths and SwissProt frequencies."""
    rng = np.random.default_rng(seed)
    lens = np.clip(rng.lognormal(np.log(median), 0.6, n).astype(int), lo, hi)
    aa = np.frombuffer(AA.encode(), np.uint8)
    seqs = rng.choice(aa, int(lens.sum()), p=FREQ / FREQ.sum())
    off = np.concatenate([[0], np.cumsum(lens)])
    return "".join(f">{prefix}{i:06d}|X\n" + bytes(seqs[off[i]:off[i + 1]]).decode() + "\n" for i in range(n))


def human_fasta() -> str:
    """The seeded human-size FASTA: 20 000 proteins, about 9.0 M residues."""
    return random_fasta(20000, 0x5A6E)


HUMAN_MODS = dict(missed_cleavages=1, static_mods={"C": 57.021464}, variable_mods={"M": [15.9949], "[": [42.010565]}, max_variable_mods=2)

SMALL = random_fasta(40, 7)
STRUCT = (">P1 first protein\nMKWVTFISLLLLFSSAYSRGVFRRDTHKSEIAHRFKDLGEEHFK\n"
          ">P2\nAAAAGGGKPEPTIDEKAAAAGGGKLLLLIIIIR\n"             # a peptide twice in one protein
          ">P3\nAAAAGGGKMMSTYSTYR\n"                             # AAAAGGGK N-terminal here, internal in P2
          ">P4\nRGVFRRDTHKSEIAHR\n"
          ">P5\nKEDITPMK\n")                                     # a short protein


def _cases() -> dict:
    c = {}
    # enzymes
    c["trypsin"] = (SMALL, dict())
    c["trypsin_missed1_static_c"] = (SMALL, dict(missed_cleavages=1, static_mods={"C": 57.021464}))
    c["aspn_nterm"] = (SMALL, dict(cleave_at="D", restrict="", c_terminal=False, missed_cleavages=1))
    c["dollar"] = (random_fasta(30, 11, median=40, lo=5, hi=60), dict(cleave_at="$", missed_cleavages=1, peptide_max_mass=9000.0))
    c["nonspecific"] = (random_fasta(12, 12, median=60, lo=10, hi=120), dict(cleave_at="", min_len=7, max_len=12, missed_cleavages=2))
    c["semi_missed0"] = (random_fasta(15, 13, median=80), dict(semi_enzymatic=True))
    c["semi_missed2"] = (random_fasta(10, 14, median=80), dict(semi_enzymatic=True, missed_cleavages=2))
    c["restrict_several"] = (SMALL, dict(cleave_at="KRE", restrict="PDE", missed_cleavages=1))
    c["cleave_non_letters"] = (SMALL, dict(cleave_at="K1r*R", restrict="p", missed_cleavages=1))
    for m in range(4):
        c[f"missed{m}_few_sites"] = (">A\nMAAAAKBBBBBWWWWWWWR\n>B\nGGGGGGGGGGGGGK\n>C\nSSSSSSSSSSSSSS\n>D\nKKKKKKKKRRRR\n", dict(missed_cleavages=m, min_len=1,
                                                                                                                          peptide_min_mass=0.0))
    # FASTA text
    c["crlf_blank_padded_split"] = ("\r\n>A desc\r\n  MKWVTFISLL \r\n\r\nLLFSSAYSRGVFRR\r\n   \r\n>B\r\nDTHKSEIAHRFKDLGEEHFK\r\n", dict(missed_cleavages=1))
    c["header_without_sequence_bare_gt"] = (">A\n>B second\nMKWVTFISLLLLFSSAYSR\n>\nGVFRRDTHKSEIAHRFK\n>C\n", dict(missed_cleavages=1))
    c["duplicate_accessions"] = (">A\nMKWVTFISLLLLFSSAYSR\n>A\nPEPTIDEKMKWVTFISLLLLFSSAYSR\n>B\nMKWVTFISLLLLFSSAYSR\n", dict(missed_cleavages=1))
    dec = ">sp|A\nMKWVTFISLLLLFSSAYSRGVFRR\n>xrev_B\nPEPTIDEKMKWVTFISLLLLFSSAYSR\n>rev_C\nRFVGRSYASSFLLLLSIFTVWKM\n>D\nPEPTIDEKLLLLR\n"
    c["tagged_generate_decoys"] = (dec, dict(missed_cleavages=1))
    c["tagged_no_generate"] = (dec, dict(missed_cleavages=1, generate_decoys=False))
    c["lowercase_and_odd_letters"] = (">A\nMKwvtfisLLLLFSSAYSRGVFRRBJOUXZ*KDTHKSEIAHRFKUOPEPTIDEK\n>B\nPEPTIDEKAAOAAUAAK\n", dict(missed_cleavages=1))
    c["bytes_over_127"] = (">A\nMKWVTF\xe9ISLLLLFSSAYSRGVFRRDTHKSEIAHRFK\n>\xc3\xa9B\nPEPTIDEKAAAAAAK\n".encode("latin-1"), dict(missed_cleavages=1))
    c["min_and_max_len"] = (">A\nMKWVK\n>B\nAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAK\n>C\nAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAK\n",
                            dict(peptide_max_mass=9000.0))
    # digest structure
    c["structure"] = (STRUCT, dict(missed_cleavages=1, min_len=1, peptide_min_mass=0.0))
    c["structure_no_generate"] = (STRUCT + ">rev_P6\nAAAAGGGKPEPTIDEKAAAAGGGK\n>rev_P7\nMKEDITPMK\n", dict(missed_cleavages=1, min_len=1, peptide_min_mass=0.0,
                                                                                          generate_decoys=False))
    c["reversal_is_target"] = (">A\nPEPTIDEKPDITPEKAMCDEFGHK\n>B\nAMCDEFGHKAFGHEDCMK\n", dict(min_len=1, peptide_min_mass=0.0))
    c["short_peptides_reversed"] = (">A\nKRAKARGGKMRCKAAAR\n", dict(min_len=1, peptide_min_mass=0.0, missed_cleavages=1))
    # modifications
    c["static_terminals"] = (SMALL, dict(missed_cleavages=1, static_mods={"C": 57.021464, "^": 1.5, "[": 42.010565, "$": 0.5, "]": 3.25, "^M": 7.0,
                                                                           "]K": 2.0}))
    c["variable_mixed"] = (SMALL, dict(missed_cleavages=1, static_mods={"C": 57.021464, "M": 1.0}, max_variable_mods=3,
                                       variable_mods={"M": [15.9949, 31.98], "[": [42.010565], "^Q": [-17.026549], "C": [-57.021464]}))
    for k in range(5):
        c[f"max_variable_mods_{k}"] = (SMALL, dict(variable_mods={"M": [15.9949], "^": [42.010565], "S": [79.966331]}, max_variable_mods=k))
    c["phospho_20_sites"] = (">A\nMSTYSTYSTYSTYSTYSTYSTYSTK\n>B\nSSSSSSSSSSTTTTTTTTTTK\n", dict(variable_mods={"S": [79.966331], "T": [79.966331], "Y": [79.966331]},
                                                                                            max_variable_mods=3, peptide_max_mass=9000.0))
    c["invalid_specs"] = (SMALL, dict(static_mods={"Z": 5.0, "": 3.0, "ABC": 2.0, "C": 57.021464, "CX": 1.0}, variable_mods={"Z": [1.0], "ABC": [2.0], "M": [15.9949]}))
    c["static_negative_zero"] = (SMALL, dict(missed_cleavages=1, static_mods={"C": -0.0, "^": -0.0, "K": 0.0}, variable_mods={"M": [-0.0], "$": [0.0]}))
    # sort and merge
    c["isobaric_il"] = (">A\nPEPTIDEKPEPTLDEKPEPTIDEKLLIIK\n>B\nPEPLIDEKIILLK\n", dict(min_len=1, peptide_min_mass=0.0, missed_cleavages=2))
    c["positional_isomers"] = (">A\nMSAMSAMSAK\n>B\nSMASMASMAK\n", dict(variable_mods={"M": [15.9949], "S": [79.966331]}, max_variable_mods=2))
    # 2 x C(32, 3) = 9 920 forms of one mass: the positional isomers of S32AK and of its reversal
    c["long_equal_mass_run"] = (">A\n" + "S" * 32 + "AK\n", dict(variable_mods={"S": [79.966331]}, max_variable_mods=3, peptide_max_mass=9000.0))
    c["mass_bounds_exact"] = (">A\nGGGGGK\n", dict(min_len=1, peptide_min_mass=0.0, peptide_max_mass=1e9))
    c["min_above_max"] = (SMALL, dict(peptide_min_mass=3000.0, peptide_max_mass=1000.0))
    c["empty_fasta"] = ("", dict())
    c["size_medium_mods"] = (random_fasta(800, 21), dict(HUMAN_MODS))
    return c


CASES = _cases()


def picked_fasta_text(seed: int, generate_decoys: bool, n_proteins: int = 60) -> str:
    """The FASTA text picked_cases.fasta_case digests (the same seeded generator, restated)."""
    rng = np.random.default_rng(seed)
    aa = np.array(list(AA))
    seqs = []
    for i in range(n_proteins):
        s = "".join(rng.choice(aa, int(rng.integers(120, 400))))
        if seqs and rng.random() < 0.5:
            src = seqs[int(rng.integers(0, len(seqs)))]
            a = int(rng.integers(0, len(src) - 60))
            s = s[:50] + src[a:a + 60] + s[50:]
        seqs.append(s)
    text = "".join(f">sp|P{i:05d}\n{s}\n" for i, s in enumerate(seqs))
    if not generate_decoys:
        text += "".join(f">rev_sp|P{i:05d}\n{s[::-1]}\n" for i, s in enumerate(seqs))
    return text


PICKED_KW = dict(missed_cleavages=1, variable_mods={"[": [42.010565]})


def _bits(a: np.ndarray) -> np.ndarray:
    b = np.ascontiguousarray(a, np.float32).view(np.uint32).copy()
    b[np.isnan(a)] = 0x7FC00000   # every NaN is None
    return b


def assert_table_equal(dev, t: dict, what: str = ""):
    """dev (sage_b200.DigestResult) == t (digest_oracle table): every array bit for bit (NaN = None), protein lists as name lists in order."""
    P = dev.peptides
    n = len(t["mono"])
    assert len(P.mono) == n, f"{what}: {len(P.mono)} peptides, oracle {n}"
    for name, a, b in (("residue_offsets", P.seq_off, t["seq_off"]), ("sequence", P.seq, t["seq"]), ("decoy", P.decoy, t["decoy"]),
                       ("missed_cleavages", P.missed, t["missed"]), ("semi_enzymatic", dev.semi_enzymatic.astype(np.uint8), t["semi"]),
                       ("modifications", _bits(P.mods), _bits(t["mods"])), ("nterm", _bits(P.nterm), _bits(t["nterm"])),
                       ("cterm", _bits(dev.cterm), _bits(t["cterm"])), ("monoisotopic", _bits(P.mono), _bits(t["mono"]))):
        a, b = np.asarray(a), np.asarray(b)
        assert a.shape == b.shape, f"{what}: {name} shape {a.shape} != {b.shape}"
        bad = np.nonzero(a != b)[0]
        assert len(bad) == 0, f"{what}: {name} differs at {len(bad)} positions, first {bad[:5].tolist()}: {a[bad[:5]].tolist()} != {b[bad[:5]].tolist()}"
    names = [x.encode("utf-8", errors="surrogateescape") for x in dev.names]
    assert names == sorted(set(names)), f"{what}: names are not distinct and in byte order"
    rank = {x: i for i, x in enumerate(names)}
    raw = t["names"].tobytes()
    no = t["name_off"]
    ids = np.array([rank.get(raw[no[j]:no[j + 1]], -1) for j in range(len(no) - 1)], np.int64)
    assert np.array_equal(dev.protein_offsets.astype(np.int64), t["prot_off"].astype(np.int64)), f"{what}: protein_offsets differ"
    assert np.array_equal(dev.protein_ids.astype(np.int64), ids), f"{what}: protein lists differ"
