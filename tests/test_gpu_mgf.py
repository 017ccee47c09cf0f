"""The MGF reader on the device (sage_b200_mgf_*, read_mgf) against the C++ oracle (oracle_mgf/) and the plain-Python restatement
(tests/mgf_reference.py): every field, every f32 bit, the ids, the precursor CSR and the info counts; str::parse::<f32> on 10^7 tokens;
the round trip of synthetic spectra; process() against process_raw and the oracle's processor; a file past 2^32 bytes; and a search
from FASTA and MGF text alone."""
import ctypes as C
import struct
from fractions import Fraction

import numpy as np
import pytest

import mgf_cases as MC
import mgf_reference as R
from oracle import oracle as O
from oracle_mgf import mgf_oracle as MO
from oracle_process import process_oracle as PO
from sage_b200 import IndexedDatabase, Scorer, SageB200Error, SpectrumProcessor, Tolerance, api, read_mgf, synth
from helpers import assert_features_equal, oracle_cfg

pytestmark = pytest.mark.gpu

EINVAL, ELIMIT = -1, -5
FIELDS = ["peak_off", "mz", "intensity", "scan_start_time", "tic", "prec_off", "prec_mz", "prec_intensity", "prec_intensity_some", "prec_charge",
          "prec_charge_some", "iso_kind", "iso_lo", "iso_hi", "id_off", "id_bytes"]
INFO = ["n_lines", "n_records", "n_spectra", "n_peaks", "n_precursors", "id_bytes", "malformed_lines", "dropped_records"]


def assert_device_equals(m, want: dict, what: str):
    assert {k: m.info[k] for k in INFO} == want["info"], what
    for k in FIELDS:
        x, y = np.ascontiguousarray(getattr(m, k)), np.ascontiguousarray(want[k])
        assert x.view(np.uint8).tobytes() == y.view(np.uint8).tobytes(), f"{what}: {k}"
    assert m.ids == [bytes(want["id_bytes"][int(a):int(b)]).decode() for a, b in zip(want["id_off"][:-1], want["id_off"][1:])]


@pytest.mark.parametrize("name", list(MC.CASES))
def test_cases_equal_oracle_and_restatement(name):
    t = MC.CASES[name]()
    m = read_mgf(t, file_id=3)
    assert m.info["file_id"] == 3 and m.info["n_bytes"] == len(t)
    assert_device_equals(m, MO.parse(t), name + " (oracle)")
    assert_device_equals(m, R.parse(t), name + " (restatement)")


@pytest.mark.parametrize("name", list(MC.ERRORS))
def test_rejected_files(name):
    t = MC.ERRORS[name]()
    with pytest.raises(SageB200Error) as e:
        read_mgf(t)
    assert e.value.code == EINVAL
    with pytest.raises(MO.MgfOracleError) as o:
        MO.parse(t)
    if name.startswith("utf8"):
        assert e.value.message.endswith(str(o.value).split("offset ")[1]), e.value.message
    else:
        assert "BEGIN IONS" in e.value.message


def _fixed_width_tokens(rng, n, n_digits, exp_lo, exp_hi):
    """n decimal tokens of n_digits random digits, a '.' at a random place, and an exponent in [exp_lo, exp_hi] written with a sign and
    a fixed width: one byte buffer and its offsets."""
    ew = len(str(max(abs(exp_lo), abs(exp_hi))))
    d = rng.integers(0, 10, (n, n_digits), dtype=np.uint8) + ord("0")
    dot = rng.integers(0, n_digits + 1, n)
    w = n_digits + 1 + 2 + ew
    buf = np.zeros((n, w), np.uint8)
    cols = np.arange(n_digits + 1)[None, :]
    src = np.where(cols < dot[:, None], cols, cols - 1)
    buf[:, :n_digits + 1] = np.where(cols == dot[:, None], ord("."), np.take_along_axis(d, np.clip(src, 0, n_digits - 1), 1))
    e = rng.integers(exp_lo, exp_hi + 1, n)
    buf[:, n_digits + 1] = ord("e")
    buf[:, n_digits + 2] = np.where(e < 0, ord("-"), ord("+"))
    a = np.abs(e)
    for k in range(ew):
        buf[:, w - 1 - k] = ord("0") + (a // 10 ** k) % 10
    return buf.tobytes(), np.arange(n + 1, dtype=np.uint64) * w


def _compare(buf: bytes, off: np.ndarray, what: str):
    n = len(off) - 1
    dev_out, dev_ok = np.zeros(n, np.float32), np.zeros(n, np.uint8)
    api._check(api.load_library().sage_b200_parse_f32(C.c_int(0), buf, api._ptr(off), C.c_uint64(n), api._ptr(dev_out), api._ptr(dev_ok)))
    ref_out, ref_ok = np.zeros(n, np.float32), np.zeros(n, np.uint8)
    MO.lib().mo_parse_f32(buf, MO._p(off), n, MO._p(ref_out), MO._p(ref_ok))
    bad = np.nonzero((dev_ok != ref_ok) | (dev_out.view(np.uint32) != ref_out.view(np.uint32)))[0]
    assert len(bad) == 0, f"{what}: {len(bad)} differ, first {buf[int(off[bad[0]]):int(off[bad[0] + 1])][:80]!r}"
    return n


def _exact_decimal(x: Fraction) -> str:
    k = 0
    while (x * 10 ** k).denominator != 1:
        k += 1
    return f"{int(x * 10 ** k)}e-{k}"


def test_parse_f32_equals_oracle_on_1e7_tokens():
    rng = np.random.default_rng(2024)
    total = 0
    for nd in range(1, 41):   # 1-40 significant digits, exponents that reach past both ends of f32
        buf, off = _fixed_width_tokens(rng, 250_000, nd, -60 - nd, 45)
        total += _compare(buf, off, f"{nd} digits")
    buf, off = _fixed_width_tokens(rng, 20_000, 800, -850, 40)   # ~800 significant digits
    total += _compare(buf, off, "800 digits")
    toks = []
    for e in ["9999999999999999999", "-9999999999999999999", "1000000000000000000", "-1000000000000000000", "18446744073709551616"]:
        toks += [f"1.5e{e}", f"0.{'0' * 30}1e{e}", f"{'9' * 30}e{e}"]
    # exact midpoints between adjacent f32s and their +-1 neighbours in the last decimal place, both signs
    for u in rng.integers(0, 0x7F7FFFFF, 20_000, dtype=np.uint64):
        a, b = np.array([u, u + 1], np.uint32).view(np.float32).astype(np.float64)
        digits, k = _exact_decimal((Fraction(float(a)) + Fraction(float(b))) / 2).split("e-")
        toks += [f"{digits}e-{k}", f"{int(digits) + 1}e-{k}", f"-{int(digits) - 1}e-{k}"]
    for u in [0, 1, 2, 0x7FFFFF, 0x800000, 0x800001, 0x7F7FFFFE, 0x7F7FFFFF]:   # subnormal, FLT_MIN and FLT_MAX edges
        x = Fraction(struct.unpack("<f", struct.pack("<I", u))[0])
        half = (Fraction(2) ** -150) if u < 0x1000000 else Fraction(2) ** ((u >> 23) - 151)
        toks += [_exact_decimal(v) for v in (x, x + half, x + half - Fraction(1, 10 ** 90), x + half + Fraction(1, 10 ** 90)) if v > 0]
    from test_mgf_reference import ACCEPT, REJECT
    toks += ACCEPT + REJECT
    bs = [t.encode() for t in toks]
    off = np.zeros(len(bs) + 1, np.uint64)
    off[1:] = np.cumsum([len(b) for b in bs])
    total += _compare(b"".join(bs), off, "edges")
    assert total >= 10_000_000
    bits, ok = api.parse_f32(ACCEPT + REJECT)
    assert ok.tolist() == [True] * len(ACCEPT) + [False] * len(REJECT)


@pytest.fixture(scope="module")
def synthetic():
    pep = synth.make_peptides(4000, seed=31, static_c=True)
    sp = synth.make_spectra(pep, 2000, seed=32)
    rt = np.random.default_rng(33).uniform(0, 7200, len(sp)).astype(np.float32)
    return pep, sp, rt, synth.write_mgf(sp, rt=rt)


def test_round_trip_synthetic(synthetic):
    _, sp, rt, text = synthetic
    m = read_mgf(text)
    assert len(m) == len(sp) and m.info["dropped_records"] == 0 and m.info["malformed_lines"] == 0
    assert np.array_equal(m.peak_off, sp.peak_off)
    assert np.array_equal(m.mz.view(np.uint32), sp.masses.view(np.uint32))
    assert np.array_equal(m.intensity.view(np.uint32), sp.intensities.view(np.uint32))
    assert np.array_equal(m.prec_mz.view(np.uint32), sp.prec_mz.view(np.uint32)) and np.array_equal(m.prec_charge, sp.prec_charge)
    want_rt = np.array([R.div60_x86(int(x)) for x in rt.view(np.uint32)], np.uint32)
    assert np.array_equal(m.scan_start_time.view(np.uint32), want_rt)
    assert m.ids == [f"synth.{i}" for i in range(len(sp))]


@pytest.mark.parametrize("kw", [dict(take_top_n=150, deisotope=False, min_deisotope_mz=0.0), dict(take_top_n=50, deisotope=True, min_deisotope_mz=131.0)])
def test_process_equals_process_raw_and_oracle(synthetic, kw):
    _, _, _, text = synthetic
    text += MC.CASES["known_answer"]().replace(b"ppm", b"Da") + MC.CASES["charges"]().replace(b"CHARGE=0", b"CHARGE=+")
    m = read_mgf(text)
    proc = SpectrumProcessor(kw["take_top_n"], kw["deisotope"], kw["min_deisotope_mz"])
    b = m.process(proc)
    raw = m.raw()
    p = proc.process_raw(raw)
    o = PO.so_process(raw, **kw)
    for got in (p.peak_off, o["peak_off"]):
        assert np.array_equal(b.peak_off, got)
    for x, y, z in ((b.masses, p.masses, o["masses"]), (b.intensities, p.intensities, o["intensities"]), (b.tic, p.tic, o["tic"])):
        assert np.array_equal(x.view(np.uint32), y.view(np.uint32)) and np.array_equal(x.view(np.uint32), np.asarray(z, np.float32).view(np.uint32))
    first = m.prec_off[:-1].astype(np.int64)
    assert np.array_equal(b.prec_mz.view(np.uint32), m.prec_mz[first].view(np.uint32)) and np.array_equal(b.prec_charge, m.first_charge())
    assert np.array_equal(b.rt.view(np.uint32), m.scan_start_time.view(np.uint32))


def test_process_rejects_charge_some_zero_and_ppm():
    m = read_mgf(MC.charges())
    with pytest.raises(SageB200Error) as e:
        m.process(SpectrumProcessor(150, False, 0.0))
    assert e.value.code == ELIMIT and "spectrum 0" in e.value.message and '"zero"' in e.value.message
    m = read_mgf(MC.known_answer())
    with pytest.raises(AssertionError):
        m.process(SpectrumProcessor(150, False, 0.0))


def test_process_raw_peak_limit():
    m = read_mgf(MC.big_spectrum())
    with pytest.raises(SageB200Error) as e:
        m.process(SpectrumProcessor(150, False, 0.0))
    assert e.value.code == ELIMIT


def test_file_past_4_gib():
    # one block of ~1 MiB, mostly a comment line the parser skips, tiled past 2^32 bytes; the last record is different
    block = b"BEGIN IONS\nTITLE=tile\nPEPMASS=500.25 7\nCHARGE=2+\n#" + b"c" * (1 << 20) + b"\n100.5 1\n200.25 2\nEND IONS\n"
    k = (1 << 32) // len(block) + 1
    last = b"BEGIN IONS\nTITLE=the last one\nPEPMASS=777.5\nRTINSECONDS=90\n300.125 4\n400.0625 8\n500 16\nEND IONS\n"
    text = block * k + last
    assert len(text) > 1 << 32
    m = read_mgf(text)
    del text
    assert m.info["n_records"] == k + 1 and len(m) == k + 1 and m.info["n_peaks"] == 2 * k + 3 and m.info["n_lines"] == 8 * k + 8
    assert m.ids[-1] == "the last one" and m.ids[0] == "tile" and m.ids[k - 1] == "tile"
    assert m.mz[-3:].tolist() == [300.125, 400.0625, 500.0] and m.intensity[-3:].tolist() == [4.0, 8.0, 16.0] and m.tic[-1] == 28.0
    assert m.prec_mz[-1] == 777.5 and m.prec_charge_some[-1] == 0 and m.scan_start_time[-1] == 1.5
    assert m.prec_off[-1] == k + 1 and m.peak_off[k] == 2 * k


def test_search_from_fasta_and_mgf_text(config1):
    # the config-1 fixture's spectrum as MGF text -> read_mgf -> process -> Scorer with config.json's parameters
    mz, it = config1["mz"], config1["intensity"]
    text = ("BEGIN IONS\nTITLE=" + config1["spectrum_id"] + "\nPEPMASS=" + str(np.float32(config1["precursor_mz"])) + "\nCHARGE="
            + str(config1["precursor_charge"]) + "+\nRTINSECONDS=" + str(np.float32(config1["scan_start_time_min"] * 60)) + "\nTOL=1\nTOLU=Da\n"
            + "".join(f"{a} {b}\n" for a, b in zip(mz.astype("U"), it.astype("U"))) + "END IONS\n")
    m = read_mgf(text)
    assert len(m) == 1 and m.ids == [config1["spectrum_id"]]
    assert np.array_equal(m.mz.view(np.uint32), mz.view(np.uint32)) and np.array_equal(m.intensity.view(np.uint32), it.view(np.uint32))
    batch = m.process(SpectrumProcessor(100, True, 0.0))
    db = IndexedDatabase.from_fasta(config1["fasta"])
    kw = dict(precursor_tol=Tolerance.ppm(-50.0, 50.0), fragment_tol=Tolerance.ppm(-10.0, 10.0), min_matched_peaks=4, min_isotope_err=-1,
              max_isotope_err=3, min_precursor_charge=2, max_precursor_charge=4, override_precursor_charge=False, max_fragment_charge=1,
              chimera=False, report_psms=1, wide_window=False, annotate_matches=False, score_type=0)
    gf, gc = Scorer(db, **kw).score_batch(batch)
    assert gc.tolist() == [1] and db.digest.peptides.sequence(int(gf[0]["peptide_idx"])) == "LQSRPAAPPAPGPGQLTLR"
    assert gf[0]["matched_peaks"] == 21
    # the oracle's processor and scorer on the oracle's parse of the same text give the same Feature rows
    o = MO.parse(text.encode())
    om, oi, ot = O.process_ms2(o["mz"], o["intensity"], int(o["prec_charge"][0]), 100, True, 0.0)
    assert np.array_equal(np.asarray(om, np.float32).view(np.uint32), batch.masses.view(np.uint32)) and np.float32(ot) == batch.tic[0]
    from helpers import oracle_db_from_peptides
    odb = oracle_db_from_peptides(db.digest.peptides)
    of, oc, _, _ = odb.score_batch(oracle_cfg(**kw), batch.as_dict())
    assert assert_features_equal(gf, gc, of, oc, 1, what="mgf end to end") == 1
