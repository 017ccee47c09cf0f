"""A plain-Python restatement of Sage's FASTA digest and database prefilter: the second CPU authority for `digest_fasta` /
`IndexedDatabase.from_fasta` (digest.cuh and the dg_* host code) and for `prefilter_fasta` (prefilter.cuh).

Written from the reference's Rust (paths relative to crates/sage/src): fasta.rs (Fasta::parse, digest, iter_chunks), enzyme.rs:33-342,
modification.rs:66-155, peptide.rs:33-388, database.rs:96-258, and the prefilter of sage-cli/src/runner.rs:104-128, 161-278. It shares no
code with oracle/ or with the device library and imports neither; the index and quick_score of the prefilter are search_reference's.

Text is handled as Rust sees it: a `str` as is, `bytes` only when valid UTF-8 (read_to_string fails otherwise: ReferenceRejects).
Sequences are the UTF-8 bytes of the protein string and every offset is a byte offset, as in Rust's `str` indexing.

Numerics: every f32 value is one np.float32 operation in Rust's order (H2O plus the residue masses as a sequential sum;
modification_mass as the sequential sum of the modifications plus nterm plus cterm; `monoisotopic += ...`). The mass filter is inclusive
and `total_cmp` is search_reference.f32_key.

Where Sage leaves an order unspecified, DESIGN.md §14 defines it:
- static mods are applied in ModificationSpecificity order, and a spec named twice keeps the last mass (HashMap::insert);
- variable mods are (spec, mass) pairs in spec order, each spec with the mass list of the last key that names it (HashMap::insert);
- `sort_unstable_by` in group_digests and `par_sort_unstable_by` in reorder_peptides are stable in emission order.

Where Sage panics, ReferencePanics is raised.
"""
from __future__ import annotations

import itertools
from dataclasses import dataclass, field

import numpy as np

import search_reference as SR

F32 = np.float32
H2O = F32(18.010565)                       # mass.rs:5
VALID_AA = b"ACDEFGHIKLMNPQRSTVWYUO"       # mass.rs:59-62
NTERM, CTERM, FULL, INTERNAL = 0, 1, 2, 3  # enzyme.rs:64-71 Position, in its derived order
PEP_N, PEP_C, PROT_N, PROT_C, RESIDUE = 0, 1, 2, 3, 4   # modification.rs:11-18 ModificationSpecificity, in its derived order
SITE_N, SITE_C = -1, -2                    # peptide.rs:335-340 Site::Nterm / Site::Cterm; Site::Sequence(i) is i
MAX_PEPS_PER_CHUNK = 1 << 23               # database.rs:143
MONO = [F32(m) for m in SR.residue_mass(np.arange(256))]   # mass.rs:70-76 per byte: 0.0 outside 'A'..='Z'


class ReferencePanics(Exception):
    """The reference panics on this input (an unwrap, an index out of bounds or an assert)."""


class ReferenceRejects(Exception):
    """The reference returns an error before digesting (the FASTA is not valid UTF-8)."""


# ------------------------------------------------------------------------------------------------ text as Rust reads it
# char::is_whitespace (Unicode White_Space), which str::trim strips; split_ascii_whitespace splits on u8::is_ascii_whitespace only.
UNICODE_WS = frozenset([*range(0x09, 0x0E), 0x20, 0x85, 0xA0, 0x1680, *range(0x2000, 0x200B), 0x2028, 0x2029, 0x202F, 0x205F, 0x3000])
ASCII_WS = frozenset(" \t\n\x0c\r")


def decode(fasta) -> str:
    if isinstance(fasta, str):
        return fasta
    try:
        return bytes(fasta).decode("utf-8")
    except UnicodeDecodeError as e:
        raise ReferenceRejects(f"not valid UTF-8: {e}") from None


def rust_lines(text: str) -> list:
    """str::lines: split_inclusive('\\n'), then strip '\\n' and one '\\r' before it (a last line without '\\n' keeps its '\\r')."""
    if not text:
        return []
    pieces = text.split("\n")
    ends = len(pieces) - 1            # pieces followed by '\n'
    if text.endswith("\n"):
        pieces.pop()
    return [p[:-1] if i < ends and p.endswith("\r") else p for i, p in enumerate(pieces)]


def rust_trim(s: str) -> str:
    a, b = 0, len(s)
    while a < b and ord(s[a]) in UNICODE_WS:
        a += 1
    while b > a and ord(s[b - 1]) in UNICODE_WS:
        b -= 1
    return s[a:b]


def first_ascii_token(s: str):
    """split_ascii_whitespace().next()."""
    i = 0
    while i < len(s) and s[i] in ASCII_WS:
        i += 1
    j = i
    while j < len(s) and s[j] not in ASCII_WS:
        j += 1
    return s[i:j] if j > i else None


# ------------------------------------------------------------------------------------------------ fasta.rs
@dataclass
class Fasta:
    targets: list          # [(accession: str, sequence: str)]
    decoy_tag: str
    generate_decoys: bool

    def iter_chunks(self, chunk_size: int):
        """fasta.rs:81-89: slice::chunks panics on 0."""
        if chunk_size == 0:
            raise ReferencePanics("chunks(0): chunk size must be non-zero")
        for i in range(0, len(self.targets), chunk_size):
            yield Fasta(self.targets[i:i + chunk_size], self.decoy_tag, self.generate_decoys)


def fasta_parse(contents, decoy_tag: str = "rev_", generate_decoys: bool = True) -> Fasta:
    """fasta.rs:14-56."""
    contents = decode(contents)
    targets = []
    last_id = ""
    s = ""

    def flush(seq):
        acc = first_ascii_token(last_id)
        if acc is None:
            raise ReferencePanics("split_ascii_whitespace().next().unwrap() on an empty header")
        if decoy_tag not in acc or not generate_decoys:
            targets.append((acc, seq))

    for line in rust_lines(contents):
        if line == "":
            continue
        line = rust_trim(line)
        if line.startswith(">"):
            if s:
                flush(s)
                s = ""
            last_id = line[1:]
        else:
            s += line
    if s:
        flush(s)
    return Fasta(targets, decoy_tag, generate_decoys)


# ------------------------------------------------------------------------------------------------ enzyme.rs
@dataclass(frozen=True)
class Enzyme:
    """enzyme.rs:124-133; `cleave` is the regex's character class (None for "$")."""
    cleave: frozenset | None
    skip_suffix: tuple
    c_terminal: bool
    semi_enzymatic: bool


def enzyme_new(cleave: str, skip_suffix: str, c_terminal: bool, semi_enzymatic: bool):
    """enzyme.rs:146-187 (`x as u8` truncates a char to its low byte, as the assert does)."""
    if not (all((ord(x) & 0xFF) in VALID_AA for x in cleave) or cleave == "$"):
        raise ReferencePanics(f"Enzyme cleavage sequence contains non-amino acid characters: {cleave}")
    if not all((ord(x) & 0xFF) in VALID_AA for x in skip_suffix):
        raise ReferencePanics(f"Enzyme cleavage restriction contains non-amino acid characters: {skip_suffix}")
    if cleave == "":
        return None
    if cleave == "$":
        return Enzyme(None, (False,) * 26, True, False)
    arr = [False] * 26
    for b in skip_suffix.encode():
        i = (b - ord("A")) & 0xFF
        if i >= 26:
            raise ReferencePanics("skip_suffix index out of bounds")
        arr[i] = True
    return Enzyme(frozenset(cleave.replace("?", "")), tuple(arr), bool(c_terminal), bool(semi_enzymatic))


@dataclass(frozen=True)
class EnzymeParameters:
    missed_cleavages: int
    min_len: int
    max_len: int
    enzyme: Enzyme | None


@dataclass
class Digest:
    decoy: bool
    semi_enzymatic: bool
    sequence: bytes
    protein: str
    missed_cleavages: int
    position: int

    def reverse(self) -> "Digest":
        """enzyme.rs:76-93 (not used by Parameters::digest; peptide.rs's test_psuedo_forward uses it)."""
        if self.decoy:
            return Digest(**self.__dict__)
        s = list(self.sequence.decode()[::-1])
        n = max(len(s) - 1, 0)
        if s:
            s[0], s[n] = s[n], s[0]
        return Digest(True, self.semi_enzymatic, "".join(s).encode(), self.protein, self.missed_cleavages, self.position)


def _matches(enzyme: Enzyme, seq: str):
    """Regex::find_iter byte ranges: the one empty match of "$" at the end, or each char of the class."""
    n = len(seq.encode())
    if enzyme.cleave is None:
        return [(n, n)]
    out, at = [], 0
    for ch in seq:
        w = len(ch.encode())
        if ch in enzyme.cleave:
            out.append((at, at + w))
        at += w
    return out


def cleavage_sites(ep: EnzymeParameters, seq: str) -> list:
    """enzyme.rs:189-217 and :221-239. A site is [start, end, missed, semi]."""
    raw = seq.encode()
    n = len(raw)
    e = ep.enzyme
    if e is None:
        return [[i, i + L, 0, False] for L in range(ep.min_len, ep.max_len + 1) for i in range(0, max(n - L, 0) + 1)]
    sites, left = [], 0
    for ms, me in _matches(e, seq):
        right = me if e.c_terminal else ms
        if right < n:
            i = (raw[right] - ord("A")) & 0xFF
            if i >= 26:
                raise ReferencePanics(f"skip_suffix[{i}] out of bounds: byte {raw[right]:#04x} after a cleavage site")
            if e.skip_suffix[i]:
                continue
        sites.append([left, right, 0, False])
        left = right
    sites.append([left, n, 0, False])
    return sites


def missed_cleavage_sites(sites: list, missed: int) -> None:
    """enzyme.rs:241-256: cleavage 1 repeats the base sites."""
    extra = []
    for c in range(1, 1 + missed + 1):
        for w in range(0, len(sites) - c + 1):
            extra.append([sites[w][0], sites[w + c - 1][1], c - 1, False])
    sites.extend(extra)


def semi_enzymatic_sites(sites: list) -> None:
    """enzyme.rs:265-287."""
    extra = []
    for start, end, missed, _ in sites:
        for cut in range(start, end):
            extra.append([start, cut, missed, True])
            extra.append([cut, end, missed, True])
    sites.extend(extra)


def is_char_boundary(raw: bytes, i: int) -> bool:
    return i == 0 or i == len(raw) or (i < len(raw) and not (0x80 <= raw[i] < 0xC0))


def enzyme_digest(ep: EnzymeParameters, seq: str, protein: str, stats: dict | None = None) -> list:
    """enzyme.rs:289-342. `stats['windows']` counts the windows that pass `sequence.get(start..end)` and the length filter (before
    `seen`)."""
    raw = seq.encode()
    n = len(raw)
    sites = cleavage_sites(ep, seq)
    missed = 0 if ep.enzyme is None else ep.missed_cleavages
    if missed > 0:
        missed_cleavage_sites(sites, missed)
    if ep.enzyme is not None and ep.enzyme.semi_enzymatic:
        semi_enzymatic_sites(sites)
    seen = set()
    out = []
    for start, end, mc, semi in sites:
        if start > end or end > n or not is_char_boundary(raw, start) or not is_char_boundary(raw, end):
            continue   # sequence.get(start..end) is None
        sub = raw[start:end]
        L = len(sub)
        position = (FULL if end == n else NTERM) if start == 0 else (CTERM if end == n else INTERNAL)
        if L >= ep.min_len and L <= ep.max_len and L > 0:
            if stats is not None:
                stats["windows"] = stats.get("windows", 0) + 1
            if sub not in seen:
                seen.add(sub)
                out.append(Digest(False, semi, sub, protein, mc, position))
    return out


def fasta_digest(f: Fasta, ep: EnzymeParameters, stats: dict | None = None) -> list:
    """fasta.rs:58-79."""
    out = []
    for protein, seq in f.targets:
        tagged = f.decoy_tag in protein
        for d in enzyme_digest(ep, seq, protein, stats):
            if tagged:
                if not f.generate_decoys:
                    d.decoy = True
                    out.append(d)
            else:
                out.append(d)
    return out


@dataclass
class DigestGroup:
    reference: Digest
    proteins: list


def group_digests(digests: list) -> list:
    """enzyme.rs:33-62; the unstable sort is taken as stable (DESIGN.md §14)."""
    if not digests:
        raise ReferencePanics("group_digests: digests[0] of an empty vector")
    digests = sorted(digests, key=lambda d: (d.position, d.decoy, d.sequence))
    groups = []
    cur = DigestGroup(digests[0], [])
    for d in digests:
        r = cur.reference
        if d.decoy == r.decoy and d.position == r.position and d.sequence == r.sequence:
            cur.proteins.append(d.protein)
        else:
            groups.append(cur)
            cur = DigestGroup(d, [d.protein])
    groups.append(cur)
    return groups


# ------------------------------------------------------------------------------------------------ modification.rs
def parse_spec(s: str):
    """ModificationSpecificity::from_str (modification.rs:66-104) as (kind, residue | -1); None where it returns an error."""
    if len(s.encode()) > 2:
        return None
    for prefix, kind in (("^", PEP_N), ("$", PEP_C), ("[", PROT_N), ("]", PROT_C)):
        if s.startswith(prefix):
            rest = s[1:]
            return (kind, (ord(rest[0]) & 0xFF) if rest else -1)
    if not s:
        return None
    c = ord(s[0]) & 0xFF
    return (RESIDUE, c) if c in VALID_AA else None


# ------------------------------------------------------------------------------------------------ peptide.rs
@dataclass
class Peptide:
    decoy: bool
    sequence: bytes
    modifications: list      # np.float32 per residue
    nterm: object            # np.float32 or None
    cterm: object
    monoisotopic: np.float32
    missed_cleavages: int
    semi_enzymatic: bool
    position: int
    proteins: list = field(default_factory=list)

    def clone(self) -> "Peptide":
        return Peptide(self.decoy, self.sequence, list(self.modifications), self.nterm, self.cterm, self.monoisotopic, self.missed_cleavages,
                       self.semi_enzymatic, self.position, list(self.proteins))

    def to_string(self) -> str:
        """peptide.rs:390-407 with integral masses (the known answers use them)."""
        fmt = lambda m: f"{float(m):+g}"  # noqa: E731
        s = f"[{fmt(self.nterm)}]-" if self.nterm is not None else ""
        for c, m in zip(self.sequence, self.modifications):
            s += chr(c) + (f"[{fmt(m)}]" if m != 0.0 else "")
        return s + (f"-[{fmt(self.cterm)}]" if self.cterm is not None else "")


def peptide_from_digest(d: Digest):
    """TryFrom<Digest> (peptide.rs:357-388); None for Err."""
    mass = H2O
    if any(c >= 128 for c in d.sequence):
        return None
    for c in d.sequence:
        m = MONO[c]
        if m == 0.0:
            return None
        mass = F32(mass + m)
    return Peptide(d.decoy, d.sequence, [F32(0.0)] * len(d.sequence), None, None, mass, d.missed_cleavages, d.semi_enzymatic, d.position,
                   [d.protein])


def modification_mass(p: Peptide) -> np.float32:
    """peptide.rs:129-133 (the sum's start, 0.0 or -0.0, only decides the sign of a zero, which `monoisotopic +=` does not see)."""
    s = F32(0.0)
    for m in p.modifications:
        s = F32(s + m)
    return F32(F32(s + (p.nterm if p.nterm is not None else F32(0.0))) + (p.cterm if p.cterm is not None else F32(0.0)))


def apply_site(p: Peptide, site: int, mass) -> None:
    """peptide.rs:136-154."""
    if site == SITE_N:
        if p.nterm is None:
            p.nterm = F32(F32(0.0) + mass)
    elif site == SITE_C:
        if p.cterm is None:
            p.cterm = F32(F32(0.0) + mass)
    elif p.modifications[site] == 0.0:
        p.modifications[site] = F32(p.modifications[site] + mass)


def _terminal_target(p: Peptide, spec):
    """The arms shared by push_resi and static_mods (peptide.rs:157-191, 211-245): the Site a terminal spec names, or None."""
    kind, r = spec
    first = p.sequence[0] if p.sequence else 0
    last = p.sequence[-1] if p.sequence else 0
    lastidx = max(len(p.sequence) - 1, 0)
    nt, ct = p.position in (NTERM, FULL), p.position in (CTERM, FULL)
    if kind == PEP_N or (kind == PROT_N and nt):
        return SITE_N if r < 0 else (0 if r == first else None)
    if kind == PEP_C or (kind == PROT_C and ct):
        return SITE_C if r < 0 else (lastidx if r == last else None)
    return None


def push_resi(p: Peptide, acc: list, spec, mass) -> None:
    """peptide.rs:156-208."""
    if spec[0] == RESIDUE:
        acc.extend((i, mass) for i, c in enumerate(p.sequence) if c == spec[1])
        return
    site = _terminal_target(p, spec)
    if site is not None:
        acc.append((site, mass))


def static_mods(p: Peptide, spec, mass) -> None:
    """peptide.rs:210-255 (a residue spec assigns, it does not add)."""
    if spec[0] == RESIDUE:
        for i, c in enumerate(p.sequence):
            if c == spec[1] and p.modifications[i] == 0.0:
                p.modifications[i] = F32(mass)
        return
    site = _terminal_target(p, spec)
    if site is not None:
        apply_site(p, site, mass)


def no_duplicates(combination) -> bool:
    """peptide.rs:321-333."""
    return sum(1 for s, _ in combination if s == SITE_N) <= 1 and sum(1 for s, _ in combination if s == SITE_C) <= 1


def same_site(combination) -> bool:
    """peptide.rs:281-286: two entries of one combination on the same Site (`continue 'next`)."""
    sites = set()
    for site, _ in combination:
        if site in sites:
            return True
        sites.add(site)
    return False


def apply(p: Peptide, variable_mods: list, static: list, combinations: int, stats: dict | None = None) -> list:
    """peptide.rs:258-305. stats['candidates'] counts the forms enumerated: the unmodified one and every combination of 1..=k sites,
    the ones no_duplicates or the same-site check skip included."""
    if not variable_mods:
        for spec, mass in static:
            static_mods(p, spec, mass)
        p.monoisotopic = F32(p.monoisotopic + modification_mass(p))
        if stats is not None:
            stats["candidates"] = stats.get("candidates", 0) + 1
        return [p]
    mods = []
    for spec, mass in variable_mods:
        push_resi(p, mods, spec, mass)
    modified = [p.clone()]
    count = 1
    for n in range(1, combinations + 1):
        for combination in itertools.combinations(mods, n):
            count += 1
            if not no_duplicates(combination) or same_site(combination):
                continue
            q = p.clone()
            for site, mass in combination:
                apply_site(q, site, mass)
            modified.append(q)
    if stats is not None:
        stats["candidates"] = stats.get("candidates", 0) + count
    for q in modified:
        for spec, mass in static:
            static_mods(q, spec, mass)
        q.monoisotopic = F32(q.monoisotopic + modification_mass(q))
    return modified


def reverse(p: Peptide) -> Peptide:
    """peptide.rs:307-318: the interior is reversed, the first and last residues stay."""
    q = p.clone()
    q.decoy = not p.decoy
    n = max(len(q.sequence) - 1, 0)
    if n > 1:
        s = bytearray(q.sequence)
        s[1:n] = s[1:n][::-1]
        q.sequence = bytes(s)
        q.modifications[1:n] = q.modifications[1:n][::-1]
    return q


def _opt_key(x):
    return (0,) if x is None else (1, float(x))


def initial_sort_key(p: Peptide):
    """peptide.rs:34-52 as a key: the sequence's bytes, then the modifications under partial_cmp (-0.0 == 0.0; finite masses only), then
    nterm and cterm with None < Some."""
    return (p.sequence, tuple(float(m) for m in p.modifications), _opt_key(p.nterm), _opt_key(p.cterm))


# ------------------------------------------------------------------------------------------------ database.rs
@dataclass
class Parameters:
    """Builder::make_parameters (database.rs:96-115) of digest_fasta's keywords."""
    enzyme: EnzymeParameters
    peptide_min_mass: np.float32
    peptide_max_mass: np.float32
    static_mods: list       # [(spec, mass)] in spec order
    variable_mods: dict     # {spec: [masses]} in spec order
    max_variable_mods: int
    decoy_tag: str
    generate_decoys: bool

    @property
    def mods(self) -> list:
        """database.rs:178-182: the flattened (spec, mass) pairs."""
        return [(s, F32(m)) for s, ms in self.variable_mods.items() for m in ms]


def make_parameters(missed_cleavages=0, min_len=5, max_len=50, cleave_at="KR", restrict="P", c_terminal=True, semi_enzymatic=False,
                    peptide_min_mass=500.0, peptide_max_mass=5000.0, static_mods=None, variable_mods=None, max_variable_mods=2,
                    decoy_tag="rev_", generate_decoys=True) -> Parameters:
    enzyme = EnzymeParameters(int(missed_cleavages), int(min_len), int(max_len), enzyme_new(cleave_at, restrict, c_terminal, semi_enzymatic))
    st: dict = {}
    for k, m in (static_mods or {}).items():   # validate_mods: HashMap::insert, the last mass of a spec wins
        s = parse_spec(k)
        if s is not None:
            st[s] = F32(m)
    var: dict = {}
    for k, ms in (variable_mods or {}).items():   # validate_var_mods: HashMap::insert, the last list of a spec wins
        s = parse_spec(k)
        if s is not None:
            var[s] = [F32(m) for m in ms]
    return Parameters(enzyme, F32(peptide_min_mass), F32(peptide_max_mass), sorted(st.items()), dict(sorted(var.items())),
                      max(int(max_variable_mods), 1), decoy_tag, bool(generate_decoys))


def auto_chunk_size(P: Parameters, f: Fasta) -> int:
    """auto_calculate_prefilter_chunk_size with prefilter_chunk_size = 0 (database.rs:142-160)."""
    total = len(fasta_digest(f, P.enzyme))
    chunk_count = (len(P.variable_mods) + 1) * (1 << P.max_variable_mods) * total // MAX_PEPS_PER_CHUNK
    return len(f.targets) if chunk_count == 0 else len(f.targets) // chunk_count


def in_mass_range(P: Parameters, mono) -> bool:
    """database.rs:201-204, inclusive at both ends."""
    return bool(mono >= P.peptide_min_mass and mono <= P.peptide_max_mass)


def digest(P: Parameters, f: Fasta, stats: dict | None = None) -> list:
    """Parameters::digest (database.rs:162-219), sequentially. stats gets windows, groups, candidates and rows (before the merge)."""
    st = {} if stats is None else stats
    st.setdefault("windows", 0)
    st.setdefault("candidates", 0)
    groups = group_digests(fasta_digest(f, P.enzyme, st))
    st["groups"] = st.get("groups", 0) + len(groups)
    mods = P.mods
    targets = {g.reference.sequence for g in groups if not g.reference.decoy}
    rows = []
    for g in groups:
        pep = peptide_from_digest(g.reference)
        if pep is None:
            continue
        pep.proteins = list(g.proteins)
        for q in apply(pep, mods, P.static_mods, P.max_variable_mods, st):
            if not in_mass_range(P, q.monoisotopic):
                continue
            for r in ([reverse(q), q] if P.generate_decoys else [q]):
                if not r.decoy or r.sequence not in targets:
                    rows.append(r)
    st["rows"] = st.get("rows", 0) + len(rows)
    reorder_peptides(rows)
    return rows


def _opt_eq(a, b) -> bool:
    return (a is None and b is None) or (a is not None and b is not None and a == b)


def reorder_peptides(rows: list) -> None:
    """database.rs:221-258: a stable sort by (total_cmp(mono), initial_sort), the adjacent merge (IEEE ==), then each protein list sorted by
    its UTF-8 bytes (String's Ord)."""
    keys = SR.f32_key(np.array([p.monoisotopic for p in rows], np.float32)).tolist()
    order = sorted(range(len(rows)), key=lambda i: (keys[i], initial_sort_key(rows[i])))
    rows[:] = [rows[i] for i in order]
    out = []
    for r in rows:
        if out:
            k = out[-1]
            if (r.monoisotopic == k.monoisotopic and r.sequence == k.sequence and len(r.modifications) == len(k.modifications)
                    and all(a == b for a, b in zip(r.modifications, k.modifications)) and _opt_eq(r.nterm, k.nterm) and _opt_eq(r.cterm, k.cterm)):
                k.proteins.extend(r.proteins)
                k.decoy = k.decoy and r.decoy
                continue
        out.append(r)
    for p in out:
        p.proteins.sort(key=lambda s: s.encode("utf-8", errors="surrogatepass"))
    rows[:] = out


# ------------------------------------------------------------------------------------------------ tables
def _nan(x) -> np.float32:
    return F32(np.nan) if x is None else F32(x)


def to_table(rows: list) -> dict:
    """The peptide table in oracle_digest's dict layout (digest_cases.assert_table_equal reads it)."""
    n = len(rows)
    seq = b"".join(p.sequence for p in rows)
    lens = np.array([len(p.sequence) for p in rows], np.int64)
    names = [a.encode("utf-8", errors="surrogatepass") for p in rows for a in p.proteins]
    return dict(seq_off=np.concatenate([[0], np.cumsum(lens)]).astype(np.uint32), seq=np.frombuffer(seq, np.uint8).copy(),
                mods=np.array([m for p in rows for m in p.modifications], np.float32).reshape(-1),
                nterm=np.array([_nan(p.nterm) for p in rows], np.float32).reshape(n), cterm=np.array([_nan(p.cterm) for p in rows], np.float32).reshape(n),
                mono=np.array([p.monoisotopic for p in rows], np.float32).reshape(n), decoy=np.array([p.decoy for p in rows], np.uint8).reshape(n),
                missed=np.array([p.missed_cleavages for p in rows], np.uint8).reshape(n), semi=np.array([p.semi_enzymatic for p in rows], np.uint8).reshape(n),
                prot_off=np.concatenate([[0], np.cumsum([len(p.proteins) for p in rows])]).astype(np.uint64),
                name_off=np.concatenate([[0], np.cumsum([len(x) for x in names])]).astype(np.uint64),
                names=np.frombuffer(b"".join(names) or b"\0", np.uint8).copy())


def digest_table(fasta, **kw):
    """(table, stats) of Parameters::digest over FASTA text with digest_fasta's keywords; stats = dict(windows, groups, candidates, rows)
    for DigestResult.info's n_windows, n_groups, n_candidates, n_rows."""
    P = make_parameters(**kw)
    f = fasta_parse(fasta, P.decoy_tag, P.generate_decoys)
    stats: dict = {}
    rows = digest(P, f, stats)
    return to_table(rows), stats


def fasta_auto_chunk_size(fasta, **kw) -> int:
    P = make_parameters(**kw)
    return auto_chunk_size(P, fasta_parse(fasta, P.decoy_tag, P.generate_decoys))


# ------------------------------------------------------------------------------------------------ the prefilter (runner.rs)
class _Arrays:
    """build_from_peptides' view of a list of Peptides."""

    def __init__(self, rows: list):
        t = to_table(rows)
        self.seq_off, self.seq, self.mods, self.nterm, self.mono = t["seq_off"], t["seq"], t["mods"], t["nterm"], t["mono"]


def prefilter(fasta, spectra, cfg: dict, chunk_size: int = 0, low_memory: bool = True, min_peaks: int = 15, bucket_size: int = 8192,
              ion_kinds=("b", "y"), min_ion_index: int = 2, **kw):
    """runner.rs:104-128 and 161-278: (table, info) with info = dict(chunk_size, n_chunks, plain_build, rows, kept), rows and kept per
    chunk. cfg holds search_reference.Scorer's keywords with the search's report_psms; the chunk scorers take report_psms + 1."""
    P = make_parameters(**kw)
    f = fasta_parse(fasta, P.decoy_tag, P.generate_decoys)
    size = auto_chunk_size(P, f) if chunk_size == 0 else int(chunk_size)
    if size >= len(f.targets):
        return to_table(digest(P, f)), dict(chunk_size=size, n_chunks=0, plain_build=1, rows=np.zeros(0, np.uint64), kept=np.zeros(0, np.uint64))
    bs = SR.next_power_of_two(bucket_size)
    scored = [s for s in SR.spectra_from_batch(spectra) if len(s.masses) >= min_peaks and s.level == 2]
    c = dict(cfg)
    c["report_psms"] = int(c.get("report_psms", 1)) + 1
    kept_rows, rows_n, kept_n = [], [], []
    for chunk in f.iter_chunks(size):
        rows = digest(P, chunk)
        db = SR.build_from_peptides(_Arrays(rows), bs, ion_kinds, min_ion_index)
        sc = SR.Scorer(db, **c)
        keep = np.zeros(len(rows), np.uint8)
        for s in scored:
            sc.quick_score(s, low_memory, keep)
        kept_rows += [r for r, k in zip(rows, keep) if k]
        rows_n.append(len(rows))
        kept_n.append(int(keep.sum()))
    reorder_peptides(kept_rows)
    return to_table(kept_rows), dict(chunk_size=size, n_chunks=len(rows_n), plain_build=0, rows=np.array(rows_n, np.uint64),
                                     kept=np.array(kept_n, np.uint64))
