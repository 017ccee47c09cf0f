"""Digest and prefilter cases aimed at the device kernels' edges, each FASTA text plus digest_fasta's keywords: cuts at the 32-residue stride
of k_dg_sites, long proteins and window limits of k_dg_windows, the compact forms of k_dg_expand up to max_variable_mods = 8, exact mass
bounds, the sort and merge, FASTA text where Rust's str handling decides, and the prefilter's chunking. Checked against the restatement
(digest_reference) and the oracle (oracle_digest)."""
from __future__ import annotations

import numpy as np

import digest_cases as DC

LOOSE = dict(min_len=1, peptide_min_mass=0.0, peptide_max_mass=1e9)


def _rand(n: int, rng, alphabet: str = "ACDEFGHILMNQSTVWY") -> str:
    """n residues without K, R or P (so the cuts and restrictions are exactly the ones placed)."""
    return "".join(rng.choice(list(alphabet), n)) if n else ""


def _stride_fasta() -> str:
    rng = np.random.default_rng(90)
    prots = []
    for L in (1, 2, 31, 32, 33, 63, 64, 65, 97):   # lengths around the 32-residue stride, each with a cut near a stride edge
        s = list(_rand(L, rng))
        for i in (L // 2, 30, 31, 32, 63):
            if i < L - 1:
                s[i] = "KR"[i % 2]
        prots.append("".join(s))
    prots.append(_rand(31, rng) + "KP" + _rand(20, rng))            # K at residue 31 (0-based), P at 32: restricted across the stride
    prots.append(_rand(30, rng) + "KPR" + _rand(20, rng))           # K at 30, P at 31 (restricted inside the stride), R at 32
    prots.append(_rand(24, rng) + "KKKKKKKKRRRRRRRR" + _rand(30, rng) + "RRRRKKKK")   # runs across strides 0/1 and at the end
    prots.append(_rand(63, rng) + "K")                              # a cut on the last residue, lane 31 of stride 1
    prots.append("KRKRKRKRKRKRKRKRKRKRKRKRKRKRKRKRKRKRKRK")        # every residue a cut (39 residues)
    prots.append("K" * 70)
    return "".join(f">S{i:02d}\n{p}\n" for i, p in enumerate(prots))


STRIDE = _stride_fasta()


def _f32_mass(seq: str) -> np.float32:
    """H2O plus the residue masses as a sequential f32 sum (peptide.rs:361-373): the mass a peptide without mods is given."""
    table = dict(zip("ACDEFGHIKLMNPQRSTVWY", [71.03711, 103.00919, 115.02694, 129.04259, 147.0684, 57.02146, 137.05891, 113.08406, 128.09496,
                                               113.08406, 131.0405, 114.04293, 97.05276, 128.05858, 156.1011, 87.03203, 101.04768, 99.06841,
                                               186.07932, 163.06332]))
    m = np.float32(18.010565)
    for c in seq:
        m = np.float32(m + np.float32(table[c]))
    return m


BOUND_FASTA = ">A\nPEPTIDEKLLSAMSGK\n>B\nMGGGGWWWK\n"
BOUND = _f32_mass("PEPTIDEK")


def _bound_cases(c: dict) -> None:
    up, down = np.nextafter(BOUND, np.float32(np.inf)), np.nextafter(BOUND, np.float32(-np.inf))
    for tag, m in (("at", BOUND), ("ulp_above", up), ("ulp_below", down)):
        c[f"mass_min_{tag}"] = (BOUND_FASTA, dict(min_len=1, peptide_min_mass=float(m), peptide_max_mass=1e9))
        c[f"mass_max_{tag}"] = (BOUND_FASTA, dict(min_len=1, peptide_min_mass=0.0, peptide_max_mass=float(m)))
    c["mass_min_eq_max"] = (BOUND_FASTA, dict(min_len=1, peptide_min_mass=float(BOUND), peptide_max_mass=float(BOUND)))


def _shared_by_many() -> str:
    rng = np.random.default_rng(91)
    # 320 proteins share LLSPEPTIDEK; accessions in descending order so the segmented id sort has work to do
    return "".join(f">Q{999 - i:04d}\nM{_rand(12, rng)}KLLSPEPTIDEK{_rand(10, rng)}R\n" for i in range(320))


def _many_accessions() -> str:
    rng = np.random.default_rng(92)
    names = [f"acc{i:05d}" for i in range(72000)]
    for i in range(0, 72000, 97):
        names[i] = f"é{i:05d}" if i % 2 else f"日本{i:05d}"           # non-ASCII accessions (two- and three-byte characters)
    order = rng.permutation(72000)
    return "".join(f">{names[j]} d\n{_rand(4, rng)}K{_rand(3, rng)}\n" for j in order)


def _multibyte_fasta() -> str:
    """20 proteins of ~100 residues with ten two-byte characters inside, none directly after a K or R (the reference panics there)."""
    rng = np.random.default_rng(93)
    out = []
    for i in range(20):
        s = list(_rand(100, rng, "ACDEFGHILMNQSTVWYKR"))
        for j in rng.choice(np.arange(5, 95), 10, replace=False):
            s[j] = "é"
            if s[j - 1] in "KR":
                s[j - 1] = "G"
        out.append(f">M{i:02d}\n{''.join(s)}\n")
    return "".join(out)


MULTIBYTE = _multibyte_fasta()
# the automatic chunk size of MULTIBYTE: (9 specs + 1) * 2^8 * windows / 2^23 is about windows / 3277, so the windows Rust skips at the
# inner byte of each character (str::get(start..end) is None) change the chunk count. The specs name U and O, which the proteins lack, so
# each chunk's digest stays one form per peptide.
MULTIBYTE_AUTO_KW = dict(cleave_at="", min_len=5, max_len=12, max_variable_mods=8,
                         variable_mods={c: [float(i + 1)] for i, c in enumerate(("U", "O", "^U", "^O", "$U", "$O", "[U", "[O", "]U"))})


def _cases() -> dict:
    c = {}
    # sites: one warp per protein, a ballot per 32-residue stride
    c["stride_trypsin"] = (STRIDE, dict(LOOSE, missed_cleavages=1))
    c["stride_trypsin_missed3"] = (STRIDE, dict(LOOSE, missed_cleavages=3))
    c["stride_nterm_cut"] = (STRIDE, dict(LOOSE, c_terminal=False, missed_cleavages=1))
    c["stride_nterm_cut_restrict_r"] = (STRIDE, dict(LOOSE, c_terminal=False, restrict="R", missed_cleavages=2))
    c["stride_semi"] = (STRIDE, dict(LOOSE, semi_enzymatic=True, missed_cleavages=1, max_len=20))
    # windows: one thread per protein
    rng = np.random.default_rng(94)
    long = ">L\n" + DC.random_fasta(1, 95, median=36000, lo=36000, hi=36000).split("\n", 1)[1]
    c["long_protein_missed3"] = (long, dict(missed_cleavages=3))
    c["long_protein_missed3_semi"] = (long, dict(missed_cleavages=3, semi_enzymatic=True, peptide_min_mass=1500.0, peptide_max_mass=1600.0))
    c["missed_above_sites"] = (">A\nMGGGGGKWWWWWWW\n>B\nMWWWWWWW\n>C\nKMWWWWK\n", dict(LOOSE, missed_cleavages=5))
    c["missed_above_sites_semi"] = (">A\nMGGGGGKWWWWWWW\n>B\nMWWWWWWW\n", dict(LOOSE, missed_cleavages=4, semi_enzymatic=True))
    ns = f">N1\n{_rand(30, rng)}\n>N2\n{_rand(50, rng)}\n>N3\n{_rand(260, rng)}\n"
    c["nonspecific_min_eq_max"] = (ns, dict(LOOSE, cleave_at="", min_len=9, max_len=9))
    c["nonspecific_above_protein"] = (ns, dict(LOOSE, cleave_at="", min_len=40, max_len=60))
    c["nonspecific_max_len_255"] = (ns, dict(LOOSE, cleave_at="", min_len=250, max_len=255))
    c["max_len_255"] = (">A\n" + _rand(254, rng) + "K" + _rand(20, rng) + "\n", dict(LOOSE, max_len=255))
    # forms: ranks to the end of the lexicographic order of up to 8 chosen sites
    phos = dict(peptide_max_mass=1e9, min_len=1, peptide_min_mass=0.0)
    c["forms_k5_20_sites"] = (">A\nG" + "S" * 20 + "K\n", dict(phos, variable_mods={"S": [79.966331]}, max_variable_mods=5))
    c["forms_k6_14_sites"] = (">A\nGST" + "SYT" * 4 + "K\n", dict(phos, variable_mods={"S": [79.966331], "T": [79.966331], "Y": [79.966331]},
                                                                 max_variable_mods=6))
    c["forms_k7_12_sites"] = (">A\nMAM" + "MS" * 5 + "K\n", dict(phos, variable_mods={"M": [15.9949], "S": [79.966331]}, max_variable_mods=7))
    c["forms_k8_8_sites"] = (">A\nGS" + "S" * 7 + "K\n>B\nGGGSSGGSGSGGSSGK\n", dict(phos, variable_mods={"S": [79.966331]}, max_variable_mods=8))
    c["forms_k2_30_sites_terminals"] = (">A\n" + "S" * 30 + "K\n", dict(phos, variable_mods={"S": [79.966331], "[": [42.010565], "$": [1.0]},
                                                                        max_variable_mods=2))
    c["two_masses_one_spec"] = (">A\nMAMGMWMK\n>B\nGMMK\n", dict(phos, variable_mods={"M": [15.9949, 31.989829]}, max_variable_mods=3))
    c["two_specs_one_residue_k4"] = (">A\nMCMCK\n", dict(phos, variable_mods={"M": [15.9949], "^M": [42.0], "C": [57.0, 58.0]}, max_variable_mods=4))
    c["nterm_competition"] = (">A\nMSTMK\n>B\nWMKMSSR\n", dict(phos, variable_mods={"^": [1.0], "[": [42.010565], "^M": [3.0]}, max_variable_mods=3))
    c["cterm_competition"] = (">A\nMSTMK\n>B\nWMKMSSK\n", dict(phos, variable_mods={"]": [5.0], "]K": [6.0], "$K": [7.0], "$": [8.0]},
                                                           max_variable_mods=3))
    c["static_and_variable_terminal"] = (">A\nMSTMK\n>B\nWMKMSSK\n", dict(phos, static_mods={"^": 5.0, "$": 2.5, "[": 11.0},
                                                                       variable_mods={"[": [42.010565], "$": [1.0], "^M": [3.0]}, max_variable_mods=2))
    c["variable_spec_repeated"] = (">A\nMCMCK\n>B\nGGCCMK\n", dict(phos, variable_mods={"C": [57.0], "CX": [58.0, 59.0], "M": [15.9949]},
                                                                 max_variable_mods=2))
    _bound_cases(c)
    # sort and merge
    c["zero_mass_forms_merge"] = (">A\nMCMCK\n>B\nGGCCMK\n", dict(phos, static_mods={"C": -0.0}, variable_mods={"M": [-0.0, 0.0], "^": [0.0]},
                                                                max_variable_mods=2))
    semi = ">P1\nGGGRGGGGAAAAWKGGG\n>P2\nGGGRAAAAWKGGG\n"    # AAAAWK: semi-enzymatic in P1, a full tryptic peptide of P2
    c["semi_flag_first_protein_wins"] = (semi, dict(LOOSE, semi_enzymatic=True))
    c["semi_flag_first_protein_wins_swapped"] = (">P0\nGGGRAAAAWKGGG\n>P1\nGGGRGGGGAAAAWKGGG\n", dict(LOOSE, semi_enzymatic=True))
    c["shared_by_320_proteins"] = (_shared_by_many(), dict(missed_cleavages=1))
    c["accessions_72000"] = (_many_accessions(), dict(LOOSE))
    # FASTA text
    c["vertical_tab_in_header"] = (">A\x0bB x\nPEPTIDEKLLLR\n>A\nPEPTIDEKMMMR\n>C\x0c\nPEPTIDEKWWWR\n", dict(LOOSE))
    c["trailing_nbsp"] = (">A\nPEPTIDEKAAAAAAR\u00a0\n>B\nMWWWWK\u3000\n>C\n\u3000GGGGK\u2009\n", dict(LOOSE, static_mods={"]": 3.0}))
    c["trailing_nbsp_no_newline"] = (">A\nPEPTIDEKAAAAAAR\u00a0", dict(LOOSE, variable_mods={"]": [3.0]}))
    # \x1c and U+200B are not White_Space: they stay in the sequence (and the header), so the last window of A and B is not a peptide
    c["whitespace_not_trimmed"] = (">A\x1c\nPEPTIDEKAAAAAAG\x1c\n>B\u0085C\nGGGKA\u200b\n", dict(LOOSE))
    c["multibyte_nonspecific"] = (MULTIBYTE, dict(LOOSE, cleave_at="", min_len=5, max_len=7))
    c["multibyte_semi"] = (MULTIBYTE, dict(LOOSE, semi_enzymatic=True, max_len=12))
    c["empty_decoy_tag_no_generate"] = (DC.STRUCT, dict(LOOSE, decoy_tag="", generate_decoys=False, missed_cleavages=1))
    return c


EDGES = _cases()

# Cases where Sage panics (its group_digests indexes an empty vector): the device and the oracle return an empty table.
EDGE_PANICS = {"empty_decoy_tag_generate": (DC.STRUCT, dict(LOOSE, decoy_tag="", generate_decoys=True))}

# Prefilter: a FASTA whose reversed decoys of one protein are targets of others, so the per-chunk decoy filter differs at every chunk size
DECOY_FASTA = (">P1\nMKADEFGHLMNKGGGGGR\n>P2\nMRANMLHGFEDKWWWWWR\n>P3\nMKADEFGHLMNKPEPTIDEKR\n>P4\nMKGGGGGRWWTTLLK\n"
               ">P5\nMRGTTLLWWKAAGGGR\n>P6\nMKPEPTIDEKSSR\n")
DECOY_KW = dict(min_len=3, peptide_min_mass=0.0)
