// sage_oracle.cpp — CPU ORACLE (TEST INFRASTRUCTURE, NOT PRODUCT CODE).
//
// A from-scratch C++17 restatement of the lazear/sage fragment-index
// search-and-score path (reference @ 0639176, v0.15.0-beta.2), written to be
// bit-faithful: every f32 product/sum is separately rounded (compile with
// -ffp-contract=off, no fast-math), comparisons follow total_cmp, sort
// stability follows the reference. It exists ONLY so that tests/,
// __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
// can check (or time) the CUDA product path against it. Nothing under
// sage_b200/ may include, link or call this file.
//
// Parity pinning: the reference cannot be compiled here (no cargo/rustc), so
// this oracle is pinned against the reference's own known-answer tests
// (tests/test_oracle_known_answers.py): Tolerance::bounds exact values
// (mass.rs:143-157), binary_search_slice cases (database.rs:569-593),
// max_fragment_charge table and Run ladder (scoring.rs:799-830), PEPTIDE ion
// tables (ion_series.rs:129-328), heap property (heap.rs:89-100),
// select_most_intense_peak (spectrum.rs:570-605), deisotope exact vectors
// (spectrum.rs:419-567), digestion order (database.rs:595-671), the
// page_search completeness property (crates/sage/tests/integration.rs:30-70)
// and the end-to-end matched_peaks==21 (crates/sage-cli/tests/integration.rs).
// Hyperscore / tie-order / chimera / open-search outputs are NOT pinned by
// any reference test ("parity unpinned" for those fields; see DESIGN.md).
//
// Each function cites the reference file:line it follows (paths relative to
// /root/reference/crates/sage/src unless stated).

#include <parallel/algorithm>
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <map>
#include <optional>
#include <set>
#include <string>
#include <unordered_set>
#include <vector>
#ifdef _OPENMP
#include <omp.h>
#endif

namespace so {

// ---------------------------------------------------------------- mass.rs:5-8
constexpr float H2O = 18.010565f;
constexpr float PROTON = 1.0072764f;
constexpr float NEUTRON = 1.00335f;

// mass.rs:64-76 (residue table) and :72-78 (monoisotopic())
static const float MONO[26] = {
    71.03711f, 0.0f,      103.00919f, 115.02694f, 129.04259f, 147.0684f, 57.02146f,
    137.05891f, 113.08406f, 0.0f,     128.09496f, 113.08406f, 131.0405f, 114.04293f,
    237.14774f, 97.05276f, 128.05858f, 156.1011f, 87.03203f,  101.04768f, 150.95363f,
    99.06841f,  186.07932f, 0.0f,     163.06332f, 0.0f};
static inline float monoisotopic(uint8_t aa) {
    return (aa >= 'A' && aa <= 'Z') ? MONO[aa - 'A'] : 0.0f;
}
static const char VALID_AA[] = "ACDEFGHIKLMNPQRSTVWYUO";  // mass.rs:59-62

// f32/f64 total_cmp as a sortable integer key (std total_cmp bit trick)
static inline int32_t f32_key(float x) {
    int32_t b;
    std::memcpy(&b, &x, 4);
    b ^= (int32_t)(((uint32_t)(b >> 31)) >> 1);
    return b;
}
static inline int total_cmp(float a, float b) {
    int32_t x = f32_key(a), y = f32_key(b);
    return x < y ? -1 : (x > y ? 1 : 0);
}
static inline int64_t f64_key(double x) {
    int64_t b;
    std::memcpy(&b, &x, 8);
    b ^= (int64_t)(((uint64_t)(b >> 63)) >> 1);
    return b;
}

// ------------------------------------------------------------ mass.rs:10-57
enum TolKind { PPM = 0, PCT = 1, DA = 2 };
struct Tolerance {
    int kind;
    float lo, hi;
    // mass.rs:21-35
    void bounds(float center, float& out_lo, float& out_hi) const {
        if (kind == PPM) {
            float dlo = center * lo / 1000000.0f;
            float dhi = center * hi / 1000000.0f;
            out_lo = center + dlo;
            out_hi = center + dhi;
        } else if (kind == PCT) {
            float dlo = center * lo / 100.0f;
            float dhi = center * hi / 100.0f;
            out_lo = center + dlo;
            out_hi = center + dhi;
        } else {
            out_lo = center + lo;
            out_hi = center + hi;
        }
    }
    // mass.rs:47-57
    Tolerance mul(float rhs) const { return Tolerance{kind, lo * rhs, hi * rhs}; }
};
// mass.rs:42-44
static inline float ppm_to_delta_mass(float center, float ppm) { return ppm * center / 1000000.0f; }

// ------------------------------------------------------- database.rs:549-561
// binary_search_slice over an abstract sorted sequence; `less_lo(i)` is
// key(slice[i], low)==Less, `le_hi(i)` is key(slice[i], high)!=Greater.
struct SearchCounters {
    uint64_t probes = 0;
};
template <class LessLo, class LeHi>
static inline void binary_search_slice(size_t n, LessLo less_lo, LeHi le_hi, size_t& left, size_t& right) {
    // partition_point(|a| key(a,&low)==Less)
    size_t lo = 0, hi = n;
    while (lo < hi) {
        size_t mid = lo + (hi - lo) / 2;
        if (less_lo(mid)) lo = mid + 1; else hi = mid;
    }
    left = lo == 0 ? 0 : lo - 1;  // saturating_sub(1)
    // slice[left..].partition_point(|a| key(a,&high)!=Greater) + left
    lo = left; hi = n;
    while (lo < hi) {
        size_t mid = lo + (hi - lo) / 2;
        if (le_hi(mid)) lo = mid + 1; else hi = mid;
    }
    right = lo;
}

// ------------------------------------------------------------ heap.rs:40-60
template <class T, class Less>
static void sift_down(T* s, size_t len, size_t index, Less less) {
    while (index * 2 + 1 < len) {
        size_t smallest = index;
        size_t l = index * 2 + 1, r = index * 2 + 2;
        if (less(s[l], s[smallest])) smallest = l;
        if (r < len && less(s[r], s[smallest])) smallest = r;
        if (smallest != index) {
            std::swap(s[smallest], s[index]);
            index = smallest;
        } else break;
    }
}
// heap.rs:7-28
template <class T, class Less>
static void bounded_min_heapify(T* s, size_t len, size_t k, Less less) {
    if (len <= k) return;
    for (size_t i = k / 2; i-- > 0;) sift_down(s, k, i, less);
    for (size_t i = k; i < len; i++) {
        if (less(s[0], s[i])) {  // slice[i] > slice[0]
            std::swap(s[i], s[0]);
            sift_down(s, k, 0, less);
        }
    }
}

// ------------------------------------------------------- ion_series.rs:8-15
enum Kind { A = 0, B = 1, C = 2, X = 3, Y = 4, Z = 5 };
static inline bool is_nterm_kind(int k) { return k <= 2; }

// --------------------------------------------------------- peptide.rs:13-31
enum Position { POS_NTERM = 0, POS_CTERM = 1, POS_FULL = 2, POS_INTERNAL = 3 };  // enzyme.rs:64-71
struct Peptide {
    bool decoy = false;
    std::string sequence;
    std::vector<float> modifications;
    std::optional<float> nterm, cterm;
    float monoisotopic = 0.0f;
    uint8_t missed_cleavages = 0;
    bool semi_enzymatic = false;
    int position = POS_INTERNAL;
    std::vector<std::string> proteins;
};

// ion_series.rs:36-85: all ions of one kind for a peptide (L-1 of them)
static void ion_series(const Peptide& p, int kind, std::vector<float>& out) {
    const float Cm = 12.0f, O = 15.994914f, H = 1.007825f, PRO = 1.0072764f, N = 14.003074f;
    const float NH3 = N + H * 2.0f + PRO;
    float nterm = p.nterm.value_or(0.0f);
    float cum;
    switch (kind) {
        case A: cum = nterm - (Cm + O); break;
        case B: cum = nterm; break;
        case C: cum = nterm + NH3; break;
        case X: cum = p.monoisotopic - nterm + (Cm + O - NH3 + N + H); break;
        case Y: cum = p.monoisotopic - nterm; break;
        default: cum = p.monoisotopic - nterm - NH3; break;
    }
    out.clear();
    size_t L = p.sequence.size();
    for (size_t idx = 0; idx + 1 < L; idx++) {
        float rm = monoisotopic((uint8_t)p.sequence[idx]) + p.modifications[idx];
        if (is_nterm_kind(kind)) cum += rm; else cum += -rm;
        out.push_back(cum);
    }
}

// ------------------------------------------------------ database.rs:367-395
struct Theoretical {
    uint32_t peptide_index;
    float fragment_mz;
};
struct DB {
    std::vector<Peptide> peptides;
    std::vector<Theoretical> fragments;
    std::vector<int> ion_kinds;
    std::vector<float> min_value;
    size_t bucket_size = 8192;
};

// ------------------------------------------------------------------ enzyme.rs
struct Digest {
    bool decoy = false;
    bool semi = false;
    std::string sequence;
    std::string protein;
    uint8_t missed = 0;
    int position = POS_INTERNAL;
};
struct EnzymeParams {
    uint8_t missed_cleavages = 0;
    size_t min_len = 5, max_len = 50;
    // enzyme (None if cleave_at == "")
    bool has_enzyme = true;
    bool dollar = false;       // cleave_at == "$"
    bool cleave[26] = {};      // regex [..] class
    bool skip_suffix[26] = {};
    bool c_terminal = true;
    bool semi_enzymatic = false;
};
struct Site { size_t start, end; uint8_t missed; bool semi; };

// enzyme.rs:145-184 (Enzyme::new)
static EnzymeParams make_enzyme(const std::string& cleave_at, const std::string& restrict_, bool c_terminal,
                                bool semi, uint8_t missed, size_t min_len, size_t max_len) {
    EnzymeParams e;
    e.missed_cleavages = missed; e.min_len = min_len; e.max_len = max_len;
    if (cleave_at.empty()) { e.has_enzyme = false; return e; }
    if (cleave_at == "$") { e.dollar = true; e.c_terminal = true; e.semi_enzymatic = false; return e; }
    for (char c : cleave_at) if (c >= 'A' && c <= 'Z') e.cleave[c - 'A'] = true;
    for (char c : restrict_) if (c >= 'A' && c <= 'Z') e.skip_suffix[c - 'A'] = true;
    e.c_terminal = c_terminal; e.semi_enzymatic = semi;
    return e;
}

// enzyme.rs:186-217 + :220-240
static std::vector<Site> cleavage_sites(const EnzymeParams& e, const std::string& seq) {
    std::vector<Site> sites;
    if (!e.has_enzyme) {
        for (size_t len = e.min_len; len <= e.max_len; len++) {
            size_t lim = seq.size() >= len ? seq.size() - len : 0;
            for (size_t i = 0; i <= lim; i++) sites.push_back({i, i + len, 0, false});
        }
        return sites;
    }
    size_t left = 0;
    auto try_site = [&](size_t right) {
        if (right < seq.size()) {
            uint8_t b = (uint8_t)seq[right];
            if (b >= 'A' && b <= 'Z' && e.skip_suffix[b - 'A']) return;
        }
        sites.push_back({left, right, 0, false});
        left = right;
    };
    if (e.dollar) {
        try_site(seq.size());  // regex "$" matches once, at end (empty match)
    } else {
        for (size_t i = 0; i < seq.size(); i++) {
            uint8_t b = (uint8_t)seq[i];
            if (b >= 'A' && b <= 'Z' && e.cleave[b - 'A']) try_site(e.c_terminal ? i + 1 : i);
        }
    }
    sites.push_back({left, seq.size(), 0, false});
    return sites;
}

// enzyme.rs:242-342
static std::vector<Digest> enzyme_digest(const EnzymeParams& e, const std::string& seq, const std::string& protein) {
    size_t n = seq.size();
    std::vector<Digest> out;
    std::vector<Site> sites = cleavage_sites(e, seq);
    uint8_t missed = e.has_enzyme ? e.missed_cleavages : 0;
    if (missed > 0) {  // :242-258
        std::vector<Site> extra;
        for (unsigned cleavage = 1; cleavage <= 1u + missed; cleavage++) {
            if (sites.size() < cleavage) continue;
            for (size_t w = 0; w + cleavage <= sites.size(); w++)
                extra.push_back({sites[w].start, sites[w + cleavage - 1].end, (uint8_t)(cleavage - 1), false});
        }
        sites.insert(sites.end(), extra.begin(), extra.end());
    }
    if (e.has_enzyme && e.semi_enzymatic) {  // :267-289
        std::vector<Site> extra;
        for (const Site& s : sites)
            for (size_t cut = s.start; cut < s.end; cut++) {
                extra.push_back({s.start, cut, s.missed, true});
                extra.push_back({cut, s.end, s.missed, true});
            }
        sites.insert(sites.end(), extra.begin(), extra.end());
    }
    std::unordered_set<std::string> seen;
    for (const Site& s : sites) {
        if (s.start > s.end || s.end > n) continue;
        // sequence.get(start..end) is None off a UTF-8 character boundary
        auto boundary = [&](size_t i) { return i == 0 || i == n || ((unsigned char)seq[i] & 0xC0) != 0x80; };
        if (!boundary(s.start) || !boundary(s.end)) continue;
        std::string sub = seq.substr(s.start, s.end - s.start);
        size_t len = sub.size();
        int pos = (s.start == 0) ? (s.end == n ? POS_FULL : POS_NTERM) : (s.end == n ? POS_CTERM : POS_INTERNAL);
        if (len >= e.min_len && len <= e.max_len && len > 0 && seen.insert(sub).second) {
            Digest d; d.sequence = sub; d.missed = s.missed; d.decoy = false; d.semi = s.semi; d.position = pos; d.protein = protein;
            out.push_back(std::move(d));
        }
    }
    return out;
}

// ------------------------------------------------------------ fasta.rs:14-56
struct Fasta {
    std::vector<std::pair<std::string, std::string>> targets;
    std::string decoy_tag;
    bool generate_decoys;
};
// char::is_whitespace: the UTF-8 byte length of the whitespace character s[0..n), 0 when s[0..n) is not one
static size_t unicode_space(const unsigned char* s, size_t n) {
    if (n == 1) return ((s[0] >= 0x09 && s[0] <= 0x0D) || s[0] == 0x20) ? 1 : 0;
    if (n == 2) return (s[0] == 0xC2 && (s[1] == 0x85 || s[1] == 0xA0)) ? 2 : 0;
    if (n != 3) return 0;
    static const char* const three[] = {"\xE1\x9A\x80", "\xE2\x80\xA8", "\xE2\x80\xA9", "\xE2\x80\xAF", "\xE2\x81\x9F", "\xE3\x80\x80"};
    if (s[0] == 0xE2 && s[1] == 0x80 && s[2] >= 0x80 && s[2] <= 0x8A) return 3;   // U+2000..U+200A
    for (const char* t : three) if (memcmp(s, t, 3) == 0) return 3;
    return 0;
}
// str::trim: Unicode whitespace at both ends
static std::string trim(const std::string& str) {
    const unsigned char* s = (const unsigned char*)str.data();
    size_t a = 0, b = str.size();
    for (bool more = true; more;) {
        more = false;
        for (size_t k = 1; k <= 3 && !more; k++) if (a + k <= b && unicode_space(s + a, k)) { a += k; more = true; }
    }
    for (bool more = true; more;) {
        more = false;
        for (size_t k = 1; k <= 3 && !more; k++) if (b >= a + k && unicode_space(s + b - k, k)) { b -= k; more = true; }
    }
    return str.substr(a, b - a);
}
// u8::is_ascii_whitespace (split_ascii_whitespace): no '\v'
static bool ascii_space(unsigned char c) { return c == ' ' || c == '\t' || c == '\n' || c == '\f' || c == '\r'; }
static Fasta fasta_parse(const std::string& contents, const std::string& decoy_tag, bool generate_decoys) {
    Fasta f; f.decoy_tag = decoy_tag; f.generate_decoys = generate_decoys;
    std::string last_id, s;
    auto flush = [&]() {
        size_t a = 0; while (a < last_id.size() && ascii_space((unsigned char)last_id[a])) a++;
        size_t b = a; while (b < last_id.size() && !ascii_space((unsigned char)last_id[b])) b++;
        std::string acc = last_id.substr(a, b - a);
        if (acc.find(decoy_tag) == std::string::npos || !generate_decoys) f.targets.push_back({acc, s});
        s.clear();
    };
    size_t pos = 0;
    while (pos <= contents.size()) {
        size_t nl = contents.find('\n', pos);
        std::string line = contents.substr(pos, nl == std::string::npos ? std::string::npos : nl - pos);
        if (!line.empty() && line.back() == '\r') line.pop_back();
        pos = nl == std::string::npos ? contents.size() + 1 : nl + 1;
        if (line.empty()) continue;
        line = trim(line);
        if (!line.empty() && line[0] == '>') {
            if (!s.empty()) flush();
            last_id = line.substr(1);
        } else {
            s += line;
        }
    }
    if (!s.empty()) flush();
    return f;
}
// fasta.rs:58-79
static std::vector<Digest> fasta_digest(const Fasta& f, const EnzymeParams& e) {
    std::vector<Digest> out;
    for (auto& t : f.targets) {
        bool tagged = t.first.find(f.decoy_tag) != std::string::npos;
        for (Digest& d : enzyme_digest(e, t.second, t.first)) {
            if (tagged) {
                if (!f.generate_decoys) { d.decoy = true; out.push_back(d); }
            } else out.push_back(d);
        }
    }
    return out;
}

// ------------------------------------------------- modification.rs:11-17,63-100
enum SpecKind { PEP_N = 0, PEP_C = 1, PROT_N = 2, PROT_C = 3, RESIDUE = 4 };
struct ModSpec {
    int kind; int residue;  // residue = -1 for None
    bool operator<(const ModSpec& o) const { return kind != o.kind ? kind < o.kind : residue < o.residue; }
};
static bool parse_modspec(const std::string& s, ModSpec& out) {
    if (s.empty() || s.size() > 2) return false;
    auto rest = [&]() { return s.size() > 1 ? (int)(uint8_t)s[1] : -1; };
    switch (s[0]) {
        case '^': out = {PEP_N, rest()}; return true;
        case '$': out = {PEP_C, rest()}; return true;
        case '[': out = {PROT_N, rest()}; return true;
        case ']': out = {PROT_C, rest()}; return true;
        default:
            if (std::strchr(VALID_AA, s[0]) && s[0] != 0) { out = {RESIDUE, (int)(uint8_t)s[0]}; return true; }
            return false;
    }
}

// ----------------------------------------------------------- peptide.rs:129-318
enum SiteKind { SITE_N = 0, SITE_C = 1, SITE_SEQ = 2 };
struct ModSite {
    int kind; uint32_t idx;
    bool operator==(const ModSite& o) const { return kind == o.kind && idx == o.idx; }
};
static float modification_mass(const Peptide& p) {  // :129-133
    float s = 0.0f;
    for (float m : p.modifications) s += m;
    return s + p.nterm.value_or(0.0f) + p.cterm.value_or(0.0f);
}
static void apply_site(Peptide& p, ModSite site, float mass) {  // :136-154
    if (site.kind == SITE_N) { if (!p.nterm) p.nterm = 0.0f + mass; }
    else if (site.kind == SITE_C) { if (!p.cterm) p.cterm = 0.0f + mass; }
    else if (p.modifications[site.idx] == 0.0f) p.modifications[site.idx] += mass;
}
static void push_resi(const Peptide& p, std::vector<std::pair<ModSite, float>>& acc, ModSpec t, float mass) {  // :156-208
    uint8_t first = p.sequence.empty() ? 0 : (uint8_t)p.sequence.front();
    uint8_t last = p.sequence.empty() ? 0 : (uint8_t)p.sequence.back();
    uint32_t lastidx = p.sequence.empty() ? 0 : (uint32_t)(p.sequence.size() - 1);
    bool nt = p.position == POS_NTERM || p.position == POS_FULL;
    bool ct = p.position == POS_CTERM || p.position == POS_FULL;
    switch (t.kind) {
        case PEP_N: if (t.residue < 0) acc.push_back({{SITE_N, 0}, mass}); else if (t.residue == first) acc.push_back({{SITE_SEQ, 0}, mass}); break;
        case PEP_C: if (t.residue < 0) acc.push_back({{SITE_C, 0}, mass}); else if (t.residue == last) acc.push_back({{SITE_SEQ, lastidx}, mass}); break;
        case PROT_N: if (nt) { if (t.residue < 0) acc.push_back({{SITE_N, 0}, mass}); else if (t.residue == first) acc.push_back({{SITE_SEQ, 0}, mass}); } break;
        case PROT_C: if (ct) { if (t.residue < 0) acc.push_back({{SITE_C, 0}, mass}); else if (t.residue == last) acc.push_back({{SITE_SEQ, lastidx}, mass}); } break;
        default:
            for (size_t i = 0; i < p.sequence.size(); i++)
                if ((uint8_t)p.sequence[i] == t.residue) acc.push_back({{SITE_SEQ, (uint32_t)i}, mass});
    }
}
static void static_mod(Peptide& p, ModSpec t, float mass) {  // :210-255
    uint8_t first = p.sequence.empty() ? 0 : (uint8_t)p.sequence.front();
    uint8_t last = p.sequence.empty() ? 0 : (uint8_t)p.sequence.back();
    uint32_t lastidx = p.sequence.empty() ? 0 : (uint32_t)(p.sequence.size() - 1);
    bool nt = p.position == POS_NTERM || p.position == POS_FULL;
    bool ct = p.position == POS_CTERM || p.position == POS_FULL;
    switch (t.kind) {
        case PEP_N: if (t.residue < 0) apply_site(p, {SITE_N, 0}, mass); else if (t.residue == first) apply_site(p, {SITE_SEQ, 0}, mass); break;
        case PEP_C: if (t.residue < 0) apply_site(p, {SITE_C, 0}, mass); else if (t.residue == last) apply_site(p, {SITE_SEQ, lastidx}, mass); break;
        case PROT_N: if (nt) { if (t.residue < 0) apply_site(p, {SITE_N, 0}, mass); else if (t.residue == first) apply_site(p, {SITE_SEQ, 0}, mass); } break;
        case PROT_C: if (ct) { if (t.residue < 0) apply_site(p, {SITE_C, 0}, mass); else if (t.residue == last) apply_site(p, {SITE_SEQ, lastidx}, mass); } break;
        default:
            for (size_t i = 0; i < p.sequence.size(); i++)
                if ((uint8_t)p.sequence[i] == t.residue && p.modifications[i] == 0.0f) p.modifications[i] = mass;
    }
}
// itertools combinations(n) over indices, lexicographic
template <class F>
static void for_combinations(size_t n_items, size_t r, F f) {
    if (r > n_items) return;
    std::vector<size_t> idx(r);
    for (size_t i = 0; i < r; i++) idx[i] = i;
    while (true) {
        f(idx);
        size_t i = r;
        while (i > 0 && idx[i - 1] == n_items - r + (i - 1)) i--;
        if (i == 0) break;
        idx[i - 1]++;
        for (size_t j = i; j < r; j++) idx[j] = idx[j - 1] + 1;
    }
}
// peptide.rs:258-305
static std::vector<Peptide> peptide_apply(Peptide self, const std::vector<std::pair<ModSpec, float>>& variable,
                                          const std::vector<std::pair<ModSpec, float>>& statics, size_t combinations) {
    if (variable.empty()) {
        for (auto& sm : statics) static_mod(self, sm.first, sm.second);
        self.monoisotopic += modification_mass(self);
        return {self};
    }
    std::vector<std::pair<ModSite, float>> mods;
    for (auto& v : variable) push_resi(self, mods, v.first, v.second);
    std::vector<Peptide> modified;
    modified.push_back(self);
    for (size_t n = 1; n <= combinations; n++) {
        for_combinations(mods.size(), n, [&](const std::vector<size_t>& idx) {
            int nn = 0, cc = 0;  // no_duplicates :321-333
            for (size_t i : idx) { if (mods[i].first.kind == SITE_N) nn++; else if (mods[i].first.kind == SITE_C) cc++; }
            if (nn > 1 || cc > 1) return;
            for (size_t a = 0; a < idx.size(); a++)
                for (size_t b = a + 1; b < idx.size(); b++)
                    if (mods[idx[a]].first == mods[idx[b]].first) return;
            Peptide p = self;
            for (size_t i : idx) apply_site(p, mods[i].first, mods[i].second);
            modified.push_back(std::move(p));
        });
    }
    for (Peptide& p : modified) {
        for (auto& sm : statics) static_mod(p, sm.first, sm.second);
        p.monoisotopic += modification_mass(p);
    }
    return modified;
}
// peptide.rs:307-318
static Peptide peptide_reverse(const Peptide& s) {
    Peptide p = s;
    p.decoy = !s.decoy;
    size_t n = p.sequence.size() == 0 ? 0 : p.sequence.size() - 1;
    if (n > 1) {
        std::reverse(p.sequence.begin() + 1, p.sequence.begin() + n);
        std::reverse(p.modifications.begin() + 1, p.modifications.begin() + n);
    }
    return p;
}
// peptide.rs:357-388
static bool peptide_from_digest(const Digest& d, Peptide& out) {
    float mass = H2O;
    for (unsigned char c : d.sequence) {
        if (c >= 128) return false;
        float m = monoisotopic(c);
        if (m == 0.0f) return false;
        mass += m;
    }
    out = Peptide();
    out.decoy = d.decoy; out.position = d.position; out.modifications.assign(d.sequence.size(), 0.0f);
    out.sequence = d.sequence; out.monoisotopic = mass; out.missed_cleavages = d.missed; out.semi_enzymatic = d.semi;
    out.proteins = {d.protein};
    return true;
}

static int cmp_optf(const std::optional<float>& a, const std::optional<float>& b) {  // Option<f32>::partial_cmp, None<Some, NaN->Equal
    if (!a && !b) return 0;
    if (!a) return -1;
    if (!b) return 1;
    return *a < *b ? -1 : (*a > *b ? 1 : 0);
}
// peptide.rs:34-52
static int initial_sort(const Peptide& a, const Peptide& b) {
    int c = a.sequence.compare(b.sequence);
    if (c) return c < 0 ? -1 : 1;
    size_t n = std::min(a.modifications.size(), b.modifications.size());
    for (size_t i = 0; i < n; i++) {
        float x = a.modifications[i], y = b.modifications[i];
        if (x < y) return -1;
        if (x > y) return 1;
        if (!(x == y)) return 0;  // partial_cmp None -> Equal
    }
    if (a.modifications.size() != b.modifications.size()) return a.modifications.size() < b.modifications.size() ? -1 : 1;
    c = cmp_optf(a.nterm, b.nterm);
    if (c) return c;
    return cmp_optf(a.cterm, b.cterm);
}

struct BuildParams {
    size_t bucket_size = 8192;
    EnzymeParams enzyme;
    float peptide_min_mass = 500.0f, peptide_max_mass = 5000.0f;
    std::vector<int> ion_kinds = {B, Y};
    size_t min_ion_index = 2;
    std::vector<std::pair<ModSpec, float>> static_mods;
    std::vector<std::pair<ModSpec, float>> variable_mods;  // flattened (spec, mass)
    size_t max_variable_mods = 2;
    std::string decoy_tag = "rev_";
    bool generate_decoys = true;
};

// database.rs:221-258
static void reorder_peptides(std::vector<Peptide>& v) {
    std::stable_sort(v.begin(), v.end(), [](const Peptide& a, const Peptide& b) {
        int c = total_cmp(a.monoisotopic, b.monoisotopic);
        if (c) return c < 0;
        return initial_sort(a, b) < 0;
    });
    std::vector<Peptide> out;
    for (Peptide& r : v) {
        if (!out.empty()) {
            Peptide& k = out.back();
            if (r.monoisotopic == k.monoisotopic && r.sequence == k.sequence && r.modifications == k.modifications &&
                r.nterm == k.nterm && r.cterm == k.cterm) {
                k.proteins.insert(k.proteins.end(), r.proteins.begin(), r.proteins.end());
                k.decoy = k.decoy && r.decoy;
                continue;
            }
        }
        out.push_back(std::move(r));
    }
    for (Peptide& p : out) std::sort(p.proteins.begin(), p.proteins.end());
    v.swap(out);
}

// enzyme.rs:33-62 (group_digests) + database.rs:162-219 (Parameters::digest)
static std::vector<Peptide> digest(const BuildParams& P, const Fasta& fasta) {
    std::vector<Digest> digests = fasta_digest(fasta, P.enzyme);
    std::vector<Peptide> out;
    if (digests.empty()) return out;
    std::stable_sort(digests.begin(), digests.end(), [](const Digest& a, const Digest& b) {
        if (a.position != b.position) return a.position < b.position;
        if (a.decoy != b.decoy) return a.decoy < b.decoy;
        return a.sequence < b.sequence;
    });
    struct Group { Digest ref; std::vector<std::string> proteins; };
    std::vector<Group> groups;
    for (const Digest& d : digests) {
        if (!groups.empty() && d.decoy == groups.back().ref.decoy && d.position == groups.back().ref.position &&
            d.sequence == groups.back().ref.sequence)
            groups.back().proteins.push_back(d.protein);
        else groups.push_back({d, {d.protein}});
    }
    std::unordered_set<std::string> targets;
    for (const Group& g : groups) if (!g.ref.decoy) targets.insert(g.ref.sequence);
    for (const Group& g : groups) {
        Peptide p;
        if (!peptide_from_digest(g.ref, p)) continue;
        p.proteins = g.proteins;
        for (Peptide& m : peptide_apply(p, P.variable_mods, P.static_mods, P.max_variable_mods)) {
            if (!(m.monoisotopic >= P.peptide_min_mass && m.monoisotopic <= P.peptide_max_mass)) continue;
            if (P.generate_decoys) {
                Peptide r = peptide_reverse(m);
                if (!r.decoy || !targets.count(r.sequence)) out.push_back(std::move(r));
            }
            if (!m.decoy || !targets.count(m.sequence)) out.push_back(std::move(m));
        }
    }
    reorder_peptides(out);
    return out;
}

// database.rs:265-365
static void build_from_peptides(DB& db, std::vector<Peptide>&& peptides, const BuildParams& P) {
    db.peptides = std::move(peptides);
    db.ion_kinds = P.ion_kinds;
    db.bucket_size = P.bucket_size;
    db.fragments.clear();
    std::vector<float> ions;
    for (size_t idx = 0; idx < db.peptides.size(); idx++) {
        const Peptide& p = db.peptides[idx];
        size_t L = p.sequence.size();
        for (int kind : P.ion_kinds) {
            ion_series(p, kind, ions);
            for (size_t ion_idx = 0; ion_idx < ions.size(); ion_idx++) {
                bool keep = is_nterm_kind(kind) ? (ion_idx + 1) > P.min_ion_index
                                                : ((L == 0 ? 0 : L - 1) - ion_idx) > P.min_ion_index;
                if (keep) db.fragments.push_back({(uint32_t)idx, ions[ion_idx]});
            }
        }
    }
    // par_sort_unstable_by fragment_mz total_cmp (rayon: parallel here too, the order is total so the result does not depend on the
    // schedule). Tie order is unobservable through page_search (pure set semantics), we use (mz, peptide) for determinism.
    __gnu_parallel::sort(db.fragments.begin(), db.fragments.end(), [](const Theoretical& a, const Theoretical& b) {
        int c = total_cmp(a.fragment_mz, b.fragment_mz);
        if (c) return c < 0;
        return a.peptide_index < b.peptide_index;
    });
    const size_t nb = (db.fragments.size() + db.bucket_size - 1) / db.bucket_size;
    db.min_value.assign(nb, 0.0f);
#pragma omp parallel for schedule(dynamic, 64)   // par_chunks_mut(bucket_size) (database.rs:337-346)
    for (long long bi = 0; bi < (long long)nb; bi++) {
        size_t s = (size_t)bi * db.bucket_size;
        size_t e = std::min(db.fragments.size(), s + db.bucket_size);
        db.min_value[bi] = db.fragments[s].fragment_mz;
        std::stable_sort(db.fragments.begin() + s, db.fragments.begin() + e,
                         [](const Theoretical& a, const Theoretical& b) { return a.peptide_index < b.peptide_index; });
    }
}

// ----------------------------------------------------------- spectrum.rs:47-79
struct Precursor {
    float mz = 0.0f;
    std::optional<uint8_t> charge;
    std::optional<Tolerance> isolation_window;
    std::optional<float> inverse_ion_mobility;
};
struct Spectrum {  // view over ProcessedSpectrum
    uint8_t level = 2;
    bool has_precursor = true;
    Precursor precursor;
    const float* masses = nullptr;
    const float* intensities = nullptr;
    size_t n_peaks = 0;
    float total_ion_current = 0.0f;
};

struct Counters {  // SURVEY.md §8(d) work counters
    uint64_t queries = 0, probes_pep = 0, probes_bucket = 0, pages = 0, probes_page = 0, entries_scanned = 0,
             candidates_scored = 0, psms = 0, matched_fragments = 0, peptide_record_floats = 0;
    void add(const Counters& o) {
        queries += o.queries; probes_pep += o.probes_pep; probes_bucket += o.probes_bucket; pages += o.pages;
        probes_page += o.probes_page; entries_scanned += o.entries_scanned; candidates_scored += o.candidates_scored;
        psms += o.psms; matched_fragments += o.matched_fragments; peptide_record_floats += o.peptide_record_floats;
    }
};
static inline uint64_t ceil_log2(size_t n) { uint64_t l = 0; while (((size_t)1 << l) < n) l++; return l; }

// spectrum.rs:134-159
static int select_most_intense_peak(const float* masses, const float* intens, size_t n, float center, Tolerance tol,
                                    std::optional<float> offset) {
    float lo, hi;
    tol.bounds(center, lo, hi);
    lo = lo + offset.value_or(0.0f);
    hi = hi + offset.value_or(0.0f);
    size_t i, j;
    binary_search_slice(n, [&](size_t k) { return total_cmp(masses[k], lo) < 0; },
                        [&](size_t k) { return total_cmp(masses[k], hi) <= 0; }, i, j);
    int best = -1;
    float max_int = 0.0f;
    for (size_t idx = i; idx < j; idx++) {
        if (masses[idx] >= lo && masses[idx] <= hi) {
            if (intens[idx] >= max_int) { max_int = intens[idx]; best = (int)idx; }
        }
    }
    return best;
}

// ----------------------------------------------------------- database.rs:402-536
struct IndexedQuery {
    const DB* db;
    float precursor_mass;
    Tolerance precursor_tol, fragment_tol;
    size_t pre_idx_lo, pre_idx_hi;
};
static IndexedQuery db_query(const DB& db, float precursor_mass, Tolerance ptol, Tolerance ftol, Counters* ctr) {
    float plo, phi;
    ptol.bounds(precursor_mass, plo, phi);
    IndexedQuery q{&db, precursor_mass, ptol, ftol, 0, 0};
    binary_search_slice(db.peptides.size(), [&](size_t k) { return total_cmp(db.peptides[k].monoisotopic, plo) < 0; },
                        [&](size_t k) { return total_cmp(db.peptides[k].monoisotopic, phi) <= 0; }, q.pre_idx_lo, q.pre_idx_hi);
    if (ctr) { ctr->queries++; ctr->probes_pep += 2 * ceil_log2(db.peptides.size()); }
    return q;
}
template <class F>
static void page_search(const IndexedQuery& q, float mass, Counters* ctr, F visit) {
    const DB& db = *q.db;
    float flo, fhi, plo, phi;
    q.fragment_tol.bounds(mass, flo, fhi);
    q.precursor_tol.bounds(q.precursor_mass, plo, phi);
    size_t left, right;
    binary_search_slice(db.min_value.size(), [&](size_t k) { return total_cmp(db.min_value[k], flo) < 0; },
                        [&](size_t k) { return total_cmp(db.min_value[k], fhi) <= 0; }, left, right);
    if (ctr) ctr->probes_bucket += 2 * ceil_log2(db.min_value.size());
    for (size_t page = left; page < right; page++) {
        size_t l = page * db.bucket_size;
        size_t r = std::min((page + 1) * db.bucket_size, db.fragments.size());
        const Theoretical* slice = db.fragments.data() + l;
        size_t n = r - l, il, ir;
        binary_search_slice(n, [&](size_t k) { return (size_t)slice[k].peptide_index < q.pre_idx_lo; },
                            [&](size_t k) { return (size_t)slice[k].peptide_index <= q.pre_idx_hi; }, il, ir);
        if (ctr) { ctr->pages++; ctr->probes_page += 2 * ceil_log2(db.bucket_size); ctr->entries_scanned += ir - il; }
        for (size_t k = il; k < ir; k++) {
            const Theoretical& f = slice[k];
            uint32_t lo32 = (uint32_t)q.pre_idx_lo, hi32 = (uint32_t)q.pre_idx_hi;
            bool ok = (f.peptide_index > lo32 || (f.peptide_index == lo32 && db.peptides[f.peptide_index].monoisotopic >= plo)) &&
                      (f.peptide_index < hi32 || (f.peptide_index == hi32 && db.peptides[f.peptide_index].monoisotopic <= phi)) &&
                      f.fragment_mz >= flo && f.fragment_mz <= fhi;
            if (ok) visit(f);
        }
    }
}

// ------------------------------------------------------------- scoring.rs
struct PreScore {  // :43-49, derived lexicographic Ord
    uint16_t matched = 0;
    uint32_t peptide = 0xFFFFFFFFu;
    uint8_t precursor_charge = 0;
    int8_t isotope_error = 0;
};
static inline bool prescore_less(const PreScore& a, const PreScore& b) {
    if (a.matched != b.matched) return a.matched < b.matched;
    if (a.peptide != b.peptide) return a.peptide < b.peptide;
    if (a.precursor_charge != b.precursor_charge) return a.precursor_charge < b.precursor_charge;
    return a.isotope_error < b.isotope_error;
}
struct InitialHits {  // :52-67
    size_t matched_peaks = 0, scored_candidates = 0;
    std::vector<PreScore> preliminary;
    void add(InitialHits&& rhs) {
        matched_peaks += rhs.matched_peaks;
        scored_candidates += rhs.scored_candidates;
        preliminary.insert(preliminary.end(), rhs.preliminary.begin(), rhs.preliminary.end());
    }
};
struct Score {  // :18-30
    uint32_t peptide = 0xFFFFFFFFu;
    uint16_t matched_b = 0, matched_y = 0;
    float summed_b = 0.0f, summed_y = 0.0f;
    size_t longest_b = 0, longest_y = 0;
    double hyperscore = 0.0;
    float ppm_difference = 0.0f;
    uint8_t precursor_charge = 0;
    int8_t isotope_error = 0;
};
struct Fragments {  // :152-161
    std::vector<int32_t> charges, kinds, fragment_ordinals;
    std::vector<float> intensities, mz_calculated, mz_experimental;
};
struct Feature {  // :69-149, numeric fields the path computes
    uint32_t peptide_idx; uint32_t peptide_len; uint32_t rank; int32_t label;
    float expmass, calcmass; uint8_t charge; float rt, ims, delta_mass, isotope_error, average_ppm;
    double hyperscore, delta_next, delta_best;
    uint32_t matched_peaks, longest_b, longest_y; float longest_y_pct; uint8_t missed_cleavages;
    float matched_intensity_pct; uint32_t scored_candidates; double poisson; float ms2_intensity;
    Fragments fragments; bool has_fragments = false;
};
struct Run {  // :771-793
    size_t start = 0, length = 0, last = 0, longest = 0;
    void matched(size_t index) {
        if (last == index) return;
        else if (start + length == index) { length += 1; longest = std::max(longest, length); }
        else { start = index; length = 1; longest = std::max(longest, length); }
        last = index;
    }
};
// :170-177
static double lnfact(uint16_t n) {
    if (n == 0) return 1.0;
    double x = (double)n;
    return x * std::log(x) - x + 0.5 * std::log(x) + 0.5 * std::log(M_PI * 2.0 * x);
}
// :179-201
static double score_type_score(int score_type, uint16_t mb, uint16_t my, float sb, float sy) {
    double s;
    if (score_type == 0) {
        double i = (double)(sb + 1.0f) * (double)(sy + 1.0f);
        s = std::log(i) + lnfact(mb) + lnfact(my);
    } else {
        float si = sb + sy;
        s = (double)log1pf(si) + lnfact(mb) + lnfact(my);
    }
    return std::isfinite(s) ? s : 255.0;
}
// :239-247
static uint8_t max_fragment_charge(int opt /* <0 = None */, uint8_t precursor_charge) {
    uint8_t m = opt >= 0 ? (uint8_t)(opt + 1) : precursor_charge;
    return std::max<uint8_t>(std::min<uint8_t>(precursor_charge, m), 2);
}

struct Scorer {  // :210-232
    const DB* db;
    Tolerance precursor_tol, fragment_tol;
    uint16_t min_matched_peaks = 4;
    int8_t min_isotope_err = 0, max_isotope_err = 0;
    uint8_t min_precursor_charge = 2, max_precursor_charge = 4;
    bool override_precursor_charge = false;
    int max_fragment_charge = -1;  // None
    bool chimera = false;
    size_t report_psms = 1;
    bool wide_window = false;
    bool annotate_matches = false;
    int score_type = 0;  // 0 Sage, 1 OpenMS

    // :322-329
    void trim_hits(InitialHits& hits) const {
        size_t len = hits.preliminary.size();
        size_t lo = std::min(report_psms * 2, len), hi = len;
        size_t k = (size_t)50 < lo ? lo : ((size_t)50 > hi ? hi : 50);  // 50.clamp(lo, hi)
        bounded_min_heapify(hits.preliminary.data(), len, k, prescore_less);
        hits.preliminary.resize(k);
    }
    // :335-382
    InitialHits matched_peaks_with_isotope(const Spectrum& q, float precursor_mass, uint8_t charge, Tolerance ptol,
                                           int8_t iso, Counters* ctr) const {
        IndexedQuery cand = db_query(*db, precursor_mass - (float)iso * NEUTRON, ptol, fragment_tol, ctr);
        uint8_t mfc = so::max_fragment_charge(max_fragment_charge, charge);
        size_t potential = cand.pre_idx_hi - cand.pre_idx_lo + 1;
        InitialHits hits;
        hits.preliminary.assign(potential, PreScore());
        for (size_t p = 0; p < q.n_peaks; p++) {
            for (uint8_t fc = 1; fc < mfc; fc++) {
                float mass = q.masses[p] * (float)fc;
                page_search(cand, mass, ctr, [&](const Theoretical& f) {
                    PreScore& sc = hits.preliminary[(size_t)f.peptide_index - cand.pre_idx_lo];
                    if (sc.matched == 0) {
                        hits.scored_candidates++;
                        sc.precursor_charge = charge;
                        sc.peptide = f.peptide_index;
                        sc.isotope_error = iso;
                    }
                    sc.matched += 1;
                    hits.matched_peaks++;
                });
            }
        }
        if (hits.matched_peaks == 0) return hits;
        trim_hits(hits);
        return hits;
    }
    // :384-416
    InitialHits matched_peaks(const Spectrum& q, float precursor_mass, uint8_t charge, Tolerance ptol, Counters* ctr) const {
        if (min_isotope_err != max_isotope_err) {
            InitialHits hits;
            for (int iso = min_isotope_err; iso <= max_isotope_err; iso++)
                hits.add(matched_peaks_with_isotope(q, precursor_mass, charge, ptol, (int8_t)iso, ctr));
            trim_hits(hits);
            return hits;
        }
        return matched_peaks_with_isotope(q, precursor_mass, charge, ptol, 0, ctr);
    }
    // :418-462
    InitialHits initial_hits(const Spectrum& q, const Precursor& pre, Counters* ctr) const {
        float mz = pre.mz - PROTON;
        InitialHits hits;
        if (wide_window) {
            for (unsigned z = min_precursor_charge; z <= max_precursor_charge; z++) {
                float pm = mz * (float)z;
                Tolerance t = pre.isolation_window.value_or(Tolerance{DA, -2.4f, 2.4f}).mul((float)z);
                hits.add(matched_peaks(q, pm, (uint8_t)z, t, ctr));
            }
        } else if (pre.charge && !override_precursor_charge) {
            uint8_t z = *pre.charge;
            hits = matched_peaks(q, mz * (float)z, z, precursor_tol, ctr);
        } else {
            for (unsigned z = min_precursor_charge; z <= max_precursor_charge; z++)
                hits.add(matched_peaks(q, mz * (float)z, (uint8_t)z, precursor_tol, ctr));
        }
        trim_hits(hits);
        return hits;
    }
    // :675-767
    Score score_candidate(const Spectrum& q, const PreScore& pre, Fragments* frags, Counters* ctr) const {
        Score score;
        score.peptide = pre.peptide; score.precursor_charge = pre.precursor_charge; score.isotope_error = pre.isotope_error;
        const Peptide& pep = db->peptides[score.peptide];
        uint8_t mfc = so::max_fragment_charge(max_fragment_charge, score.precursor_charge);
        Run b_run, y_run;
        static thread_local std::vector<float> ions;   // the reference's IonSeries is an iterator: no allocation per candidate
        if (ctr) { ctr->candidates_scored++; ctr->peptide_record_floats += 2 * pep.sequence.size() + 2; }
        for (int kind : db->ion_kinds) {
            ion_series(pep, kind, ions);
            for (size_t idx = 0; idx < ions.size(); idx++) {
                for (uint8_t fc = 1; fc < mfc; fc++) {
                    float mz = ions[idx] / (float)fc;
                    int pk = select_most_intense_peak(q.masses, q.intensities, q.n_peaks, mz, fragment_tol, std::nullopt);
                    if (pk < 0) continue;
                    float peak_mass = q.masses[pk], peak_int = q.intensities[pk];
                    score.ppm_difference += peak_int * std::fabs(mz - peak_mass) * 2E6f / (mz + peak_mass);
                    float exp_mz = peak_mass + PROTON, calc_mz = mz + PROTON;
                    if (is_nterm_kind(kind)) { score.matched_b += 1; score.summed_b += peak_int; b_run.matched(idx); }
                    else { score.matched_y += 1; score.summed_y += peak_int; y_run.matched(idx); }
                    if (frags) {
                        int32_t ord = is_nterm_kind(kind) ? (int32_t)idx + 1
                                                          : (int32_t)(pep.sequence.empty() ? 0 : pep.sequence.size() - 1) - (int32_t)idx;
                        frags->kinds.push_back(kind); frags->charges.push_back(fc);
                        frags->mz_experimental.push_back(exp_mz); frags->mz_calculated.push_back(calc_mz);
                        frags->fragment_ordinals.push_back(ord); frags->intensities.push_back(peak_int);
                    }
                }
            }
        }
        score.hyperscore = score_type_score(score_type, score.matched_b, score.matched_y, score.summed_b, score.summed_y);
        score.longest_b = b_run.longest; score.longest_y = y_run.longest;
        score.ppm_difference /= score.summed_b + score.summed_y;
        return score;
    }
    // :478-595
    void build_features(const Spectrum& q, const Precursor& pre, const InitialHits& hits, size_t report,
                        std::vector<Feature>& features, Counters* ctr) const {
        struct SV { Score s; Fragments f; };
        std::vector<SV> sv;
        for (const PreScore& p : hits.preliminary) {
            if (p.peptide == 0xFFFFFFFFu) continue;
            SV e;
            e.s = score_candidate(q, p, annotate_matches ? &e.f : nullptr, ctr);
            if ((unsigned)(e.s.matched_b + e.s.matched_y) >= min_matched_peaks) sv.push_back(std::move(e));
        }
        std::stable_sort(sv.begin(), sv.end(), [](const SV& a, const SV& b) { return f64_key(b.s.hyperscore) < f64_key(a.s.hyperscore); });
        double lambda = (double)hits.matched_peaks / (double)hits.scored_candidates;
        float mz = pre.mz - PROTON;
        for (size_t idx = 0; idx < std::min(report, sv.size()); idx++) {
            const Score& s = sv[idx].s;
            const Peptide& pep = db->peptides[s.peptide];
            float precursor_mass = mz * (float)s.precursor_charge;
            double next = idx + 1 < sv.size() ? sv[idx + 1].s.hyperscore : 0.0;
            double best = sv[0].s.hyperscore;
            uint16_t k = (uint16_t)(s.matched_b + s.matched_y);
            double log10_poisson = ((double)k * std::log(lambda) - lambda - lnfact(k)) / M_LN10;
            float iso = (float)s.isotope_error * NEUTRON;
            float delta_mass = (precursor_mass - pep.monoisotopic - iso) * 2E6f / (precursor_mass - iso + pep.monoisotopic);
            Feature f;
            f.peptide_idx = s.peptide; f.peptide_len = (uint32_t)pep.sequence.size(); f.rank = (uint32_t)idx + 1;
            f.label = pep.decoy ? -1 : 1; f.expmass = precursor_mass; f.calcmass = pep.monoisotopic; f.charge = s.precursor_charge;
            f.rt = 0.0f; f.ims = pre.inverse_ion_mobility.value_or(0.0f);
            f.delta_mass = delta_mass; f.isotope_error = iso; f.average_ppm = s.ppm_difference;
            f.hyperscore = s.hyperscore; f.delta_next = s.hyperscore - next; f.delta_best = best - s.hyperscore;
            f.matched_peaks = k; f.matched_intensity_pct = 100.0f * (s.summed_b + s.summed_y) / q.total_ion_current;
            f.poisson = std::isfinite(log10_poisson) ? log10_poisson : -INFINITY;
            f.longest_b = (uint32_t)s.longest_b; f.longest_y = (uint32_t)s.longest_y;
            f.longest_y_pct = (float)s.longest_y / (float)pep.sequence.size();
            f.scored_candidates = (uint32_t)hits.scored_candidates; f.missed_cleavages = pep.missed_cleavages;
            f.ms2_intensity = s.summed_b + s.summed_y;
            if (annotate_matches) { f.fragments = std::move(sv[idx].f); f.has_fragments = true; }
            features.push_back(std::move(f));
            if (ctr) ctr->psms++;
        }
    }
    // :465-474
    std::vector<Feature> score_standard(const Spectrum& q, Counters* ctr) const {
        InitialHits hits = initial_hits(q, q.precursor, ctr);
        std::vector<Feature> out;
        build_features(q, q.precursor, hits, report_psms, out, ctr);
        return out;
    }
    // :598-644
    void remove_matched_peaks(std::vector<float>& masses, std::vector<float>& intens, float& tic, const Feature& psm) const {
        const Peptide& pep = db->peptides[psm.peptide_idx];
        uint8_t mfc = so::max_fragment_charge(max_fragment_charge, psm.charge);
        std::vector<std::pair<float, float>> to_remove;
        std::vector<float> ions;
        for (int kind : db->ion_kinds) {
            ion_series(pep, kind, ions);
            for (float frag : ions)
                for (uint8_t fc = 1; fc < mfc; fc++) {
                    int pk = select_most_intense_peak(masses.data(), intens.data(), masses.size(), frag / (float)fc, fragment_tol, std::nullopt);
                    if (pk >= 0) to_remove.push_back({masses[pk], intens[pk]});
                }
        }
        std::vector<float> m2, i2;
        for (size_t i = 0; i < masses.size(); i++) {
            bool rm = false;
            for (auto& tr : to_remove) if (tr.first == masses[i] && tr.second == intens[i]) { rm = true; break; }
            if (!rm) { m2.push_back(masses[i]); i2.push_back(intens[i]); }
        }
        masses.swap(m2); intens.swap(i2);
        float s = 0.0f;
        for (float x : intens) s += x;
        tic = s;
    }
    // :648-672
    std::vector<Feature> score_chimera_fast(const Spectrum& q0, Counters* ctr) const {
        std::vector<float> masses(q0.masses, q0.masses + q0.n_peaks), intens(q0.intensities, q0.intensities + q0.n_peaks);
        Spectrum q = q0;
        InitialHits hits = initial_hits(q, q.precursor, ctr);
        std::vector<Feature> cands;
        size_t prev = 0;
        while (cands.size() < report_psms) {
            q.masses = masses.data(); q.intensities = intens.data(); q.n_peaks = masses.size();
            build_features(q, q.precursor, hits, 1, cands, ctr);
            if (cands.size() > prev) {
                remove_matched_peaks(masses, intens, q.total_ion_current, cands[prev]);
                cands[prev].rank = (uint32_t)prev + 1;
                prev = cands.size();
            } else break;
        }
        return cands;
    }
    // :255-298 quick_score (prefilter). `keep` has one byte per peptide.
    // The low-memory branch calls bounded_min_heapify on Vec<Score>; heap.rs compares with `<` / `>`, i.e. Score's DERIVED PartialOrd
    // (lexicographic, first field = peptide, scoring.rs:17-30), not its hyperscore Ord — restated literally.
    int quick_score(const Spectrum& q, bool low_memory, uint8_t* keep) const {
        if (q.level != 2) return -1;
        if (!q.has_precursor) return -2;
        InitialHits hits = initial_hits(q, q.precursor, nullptr);
        if (low_memory) {
            std::vector<Score> sv;
            for (const PreScore& p : hits.preliminary) {
                if (p.peptide == 0xFFFFFFFFu) continue;
                Score sc = score_candidate(q, p, nullptr, nullptr);
                if ((unsigned)(sc.matched_b + sc.matched_y) < min_matched_peaks) continue;
                sv.push_back(sc);
            }
            size_t k = std::min(report_psms, sv.size());
            auto lt = [](const Score& a, const Score& b) {  // derived PartialOrd::lt; a NaN field makes the comparison false
                if (a.peptide != b.peptide) return a.peptide < b.peptide;
                if (a.matched_b != b.matched_b) return a.matched_b < b.matched_b;
                if (a.matched_y != b.matched_y) return a.matched_y < b.matched_y;
                if (!(a.summed_b == b.summed_b)) return a.summed_b < b.summed_b;
                if (!(a.summed_y == b.summed_y)) return a.summed_y < b.summed_y;
                if (a.longest_b != b.longest_b) return a.longest_b < b.longest_b;
                if (a.longest_y != b.longest_y) return a.longest_y < b.longest_y;
                if (!(a.hyperscore == b.hyperscore)) return a.hyperscore < b.hyperscore;
                if (!(a.ppm_difference == b.ppm_difference)) return a.ppm_difference < b.ppm_difference;
                if (a.precursor_charge != b.precursor_charge) return a.precursor_charge < b.precursor_charge;
                return a.isotope_error < b.isotope_error;
            };
            bounded_min_heapify(sv.data(), sv.size(), k, lt);
            for (size_t i = 0; i < k; i++) keep[sv[i].peptide] = 1;
        } else {
            for (const PreScore& p : hits.preliminary)
                if (p.peptide != 0xFFFFFFFFu) keep[p.peptide] = 1;
        }
        return 0;
    }
    // :300-309. Returns -1 (reference panics) for non-MS2 / missing precursor.
    int score(const Spectrum& q, std::vector<Feature>& out, Counters* ctr) const {
        if (q.level != 2) return -1;
        if (!q.has_precursor) return -2;
        out = chimera ? score_chimera_fast(q, ctr) : score_standard(q, ctr);
        return 0;
    }
};

// --------------------------------------------------------- spectrum.rs:179-239
struct Deisotoped { float mz, intensity; int charge /* -1 None */; int64_t envelope /* -1 None */; };
static std::vector<Deisotoped> deisotope(const float* mz, const float* inten, size_t n, uint8_t max_charge, float ppm, float min_mz) {
    std::vector<Deisotoped> peaks(n);
    for (size_t i = 0; i < n; i++) peaks[i] = {mz[i], inten[i], -1, -1};
    for (size_t i = n; i-- > 0;) {
        size_t j = i == 0 ? 0 : i - 1;
        while (mz[i] - mz[j] <= NEUTRON + ppm_to_delta_mass(mz[i], ppm) && mz[j] >= min_mz) {
            float delta = mz[i] - mz[j];
            float tol = ppm_to_delta_mass(mz[i], ppm);
            for (unsigned charge = 1; charge <= max_charge; charge++) {
                float iso = NEUTRON / (float)charge;
                if (std::fabs(delta - iso) <= tol && inten[i] < inten[j]) {
                    if (peaks[i].charge >= 0 && peaks[i].charge != (int)charge) continue;
                    peaks[j].intensity += peaks[i].intensity;
                    peaks[j].charge = (int)charge;
                    peaks[i].charge = (int)charge;
                    peaks[i].envelope = (int64_t)j;
                }
            }
            j = j == 0 ? 0 : j - 1;
            if (j == 0) break;
        }
    }
    return peaks;
}
static void path_compression(std::vector<Deisotoped>& peaks) {  // :230-239
    for (size_t i = 0; i < peaks.size(); i++) {
        if (peaks[i].envelope >= 0) {
            int64_t up = peaks[(size_t)peaks[i].envelope].envelope;
            if (up >= 0) peaks[i].envelope = up;
            peaks[i].intensity = 0.0f;
        }
    }
}
struct Peak { float intensity, mass; };
// spectrum.rs:279-336 + :380-412 (MS2 branch of SpectrumProcessor::process)
static void process_ms2(const float* mz, const float* inten, size_t n, int precursor_charge /* <=0 None */, size_t take_top_n,
                        bool do_deisotope, float min_deisotope_mz, std::vector<float>& masses, std::vector<float>& intens, float& tic) {
    uint8_t charge = precursor_charge > 0 ? (uint8_t)precursor_charge : 3;
    std::vector<Peak> peaks;
    if (do_deisotope) {
        std::vector<Deisotoped> d = deisotope(mz, inten, n, charge, 10.0f, min_deisotope_mz);
        std::stable_sort(d.begin(), d.end(), [](const Deisotoped& a, const Deisotoped& b) {
            int c = total_cmp(b.intensity, a.intensity);
            if (c) return c < 0;
            return total_cmp(a.mz, b.mz) < 0;
        });
        for (const Deisotoped& p : d) {
            if (p.envelope >= 0) continue;
            if (peaks.size() >= take_top_n) break;
            float mass = (p.mz - PROTON) * (float)(p.charge >= 0 ? p.charge : 1);
            peaks.push_back({p.intensity, mass});
        }
    } else {
        for (size_t i = 0; i < n; i++) peaks.push_back({inten[i], (mz[i] - PROTON) * 1.0f});
        auto less = [](const Peak& a, const Peak& b) {
            int c = total_cmp(a.intensity, b.intensity);
            if (c) return c < 0;
            return total_cmp(a.mass, b.mass) < 0;
        };
        bounded_min_heapify(peaks.data(), peaks.size(), take_top_n, less);
        if (peaks.size() > take_top_n) peaks.resize(take_top_n);
    }
    std::stable_sort(peaks.begin(), peaks.end(), [](const Peak& a, const Peak& b) { return total_cmp(a.mass, b.mass) < 0; });
    masses.clear(); intens.clear();
    float s = 0.0f;
    for (const Peak& p : peaks) { masses.push_back(p.mass); intens.push_back(p.intensity); }
    for (float x : intens) s += x;
    tic = s;
}

}  // namespace so

// =============================================================== C API (ctypes)
using namespace so;

extern "C" {

struct so_tol { int32_t kind; float lo, hi; };
struct so_scorer_params {
    so_tol precursor_tol, fragment_tol;
    uint16_t min_matched_peaks; int8_t min_isotope_err, max_isotope_err;
    uint8_t min_precursor_charge, max_precursor_charge, override_precursor_charge; int8_t max_fragment_charge /* <0 None */;
    uint8_t chimera, wide_window, annotate_matches, score_type;
    uint32_t report_psms;
};
struct so_feature {
    uint32_t spectrum, peptide_idx, peptide_len, rank; int32_t label;
    float expmass, calcmass; uint32_t charge; float delta_mass, isotope_error, average_ppm;
    double hyperscore, delta_next, delta_best;
    uint32_t matched_peaks, longest_b, longest_y; float longest_y_pct; uint32_t missed_cleavages;
    float matched_intensity_pct; uint32_t scored_candidates; double poisson; float ms2_intensity; uint32_t frag_offset, frag_count;
};
struct so_fragment { int32_t kind, charge, ordinal; float intensity, mz_calculated, mz_experimental; };
struct so_counters { uint64_t queries, probes_pep, probes_bucket, pages, probes_page, entries_scanned, candidates_scored, psms, peptide_record_floats; };

struct so_build_params {
    uint64_t bucket_size; uint8_t missed_cleavages; uint64_t min_len, max_len;
    const char* cleave_at; const char* restrict_; uint8_t c_terminal, semi_enzymatic;
    float peptide_min_mass, peptide_max_mass;
    const uint8_t* ion_kinds; uint64_t n_kinds; uint64_t min_ion_index;
    const char* const* static_mod_specs; const float* static_mod_masses; uint64_t n_static;
    const char* const* var_mod_specs; const float* var_mod_masses; uint64_t n_var;
    uint64_t max_variable_mods; const char* decoy_tag; uint8_t generate_decoys;
};

static BuildParams to_build_params(const so_build_params* p) {
    BuildParams P;
    // Builder::make_parameters database.rs:96-115
    size_t bs = (size_t)p->bucket_size, pw = 1;
    while (pw < bs) pw <<= 1;
    P.bucket_size = pw;
    P.enzyme = make_enzyme(p->cleave_at ? p->cleave_at : "", p->restrict_ ? p->restrict_ : "", p->c_terminal, p->semi_enzymatic,
                           p->missed_cleavages, (size_t)p->min_len, (size_t)p->max_len);
    P.peptide_min_mass = p->peptide_min_mass; P.peptide_max_mass = p->peptide_max_mass;
    P.ion_kinds.clear();
    for (uint64_t i = 0; i < p->n_kinds; i++) P.ion_kinds.push_back(p->ion_kinds[i]);
    P.min_ion_index = (size_t)p->min_ion_index;
    std::map<ModSpec, float> st;
    for (uint64_t i = 0; i < p->n_static; i++) { ModSpec m; if (parse_modspec(p->static_mod_specs[i], m)) st[m] = p->static_mod_masses[i]; }
    for (auto& kv : st) P.static_mods.push_back(kv);
    std::vector<std::pair<ModSpec, float>> var;
    // validate_var_mods (modification.rs:129-155) is HashMap::insert per spec string: a later string naming the same spec replaces the masses
    // of the earlier one (entries with equal strings are one string's list)
    std::vector<std::string> var_str;
    for (uint64_t i = 0; i < p->n_var; i++) {
        ModSpec m;
        if (!parse_modspec(p->var_mod_specs[i], m)) continue;
        for (size_t j = 0; j < var.size();) {
            if (!(var[j].first < m) && !(m < var[j].first) && var_str[j] != p->var_mod_specs[i]) { var.erase(var.begin() + j); var_str.erase(var_str.begin() + j); }
            else j++;
        }
        var.push_back({m, p->var_mod_masses[i]});
        var_str.push_back(p->var_mod_specs[i]);
    }
    std::stable_sort(var.begin(), var.end(), [](auto& a, auto& b) { return a.first < b.first; });
    P.variable_mods = var;
    P.max_variable_mods = std::max<size_t>((size_t)p->max_variable_mods, 1);
    P.decoy_tag = p->decoy_tag ? p->decoy_tag : "rev_";
    P.generate_decoys = p->generate_decoys;
    return P;
}

void* so_db_from_fasta(const char* fasta_text, const so_build_params* p) {
    BuildParams P = to_build_params(p);
    // read_fasta(path, decoy_tag, generate_decoys) sage-cloudpath/src/util.rs:121
    Fasta f = fasta_parse(fasta_text, P.decoy_tag, P.generate_decoys);
    DB* db = new DB();
    build_from_peptides(*db, digest(P, f), P);
    return db;
}

// Peptides supplied already in final (sorted, deduplicated) order.
void* so_db_from_peptides(uint64_t n_pep, const uint32_t* seq_off, const uint8_t* seq, const float* mods, const float* nterm /*NaN=None*/,
                          const float* mono, const uint8_t* decoy, const uint8_t* missed, uint64_t bucket_size, const uint8_t* kinds,
                          uint64_t n_kinds, uint64_t min_ion_index) {
    std::vector<Peptide> peps(n_pep);
    for (uint64_t i = 0; i < n_pep; i++) {
        Peptide& p = peps[i];
        p.sequence.assign((const char*)seq + seq_off[i], seq_off[i + 1] - seq_off[i]);
        p.modifications.assign(mods + seq_off[i], mods + seq_off[i + 1]);
        if (!std::isnan(nterm[i])) p.nterm = nterm[i];
        p.monoisotopic = mono[i]; p.decoy = decoy[i]; p.missed_cleavages = missed[i];
    }
    BuildParams P;
    P.bucket_size = (size_t)bucket_size;
    P.ion_kinds.clear();
    for (uint64_t i = 0; i < n_kinds; i++) P.ion_kinds.push_back(kinds[i]);
    P.min_ion_index = (size_t)min_ion_index;
    DB* db = new DB();
    build_from_peptides(*db, std::move(peps), P);
    return db;
}
void so_db_free(void* h) { delete (DB*)h; }
uint64_t so_db_n_peptides(void* h) { return ((DB*)h)->peptides.size(); }
uint64_t so_db_n_fragments(void* h) { return ((DB*)h)->fragments.size(); }
uint64_t so_db_n_buckets(void* h) { return ((DB*)h)->min_value.size(); }
uint64_t so_db_bucket_size(void* h) { return ((DB*)h)->bucket_size; }
uint64_t so_db_total_residues(void* h) { uint64_t s = 0; for (auto& p : ((DB*)h)->peptides) s += p.sequence.size(); return s; }
void so_db_export(void* h, uint32_t* frag_pep, float* frag_mz, float* bucket_min, float* pep_mono, uint32_t* seq_off, uint8_t* seq, float* mods,
                  float* nterm, float* cterm, uint8_t* decoy, uint8_t* missed) {
    DB* db = (DB*)h;
    for (size_t i = 0; i < db->fragments.size(); i++) { frag_pep[i] = db->fragments[i].peptide_index; frag_mz[i] = db->fragments[i].fragment_mz; }
    for (size_t i = 0; i < db->min_value.size(); i++) bucket_min[i] = db->min_value[i];
    uint32_t off = 0;
    for (size_t i = 0; i < db->peptides.size(); i++) {
        const Peptide& p = db->peptides[i];
        pep_mono[i] = p.monoisotopic; seq_off[i] = off;
        std::memcpy(seq + off, p.sequence.data(), p.sequence.size());
        std::memcpy(mods + off, p.modifications.data(), 4 * p.modifications.size());
        off += (uint32_t)p.sequence.size();
        nterm[i] = p.nterm ? *p.nterm : NAN; cterm[i] = p.cterm ? *p.cterm : NAN;
        decoy[i] = p.decoy; missed[i] = p.missed_cleavages;
    }
    seq_off[db->peptides.size()] = off;
}
// Display form of a peptide (peptide.rs:390-407) for the digestion known-answer test. Mods printed with %+g.
int so_db_peptide_string(void* h, uint64_t i, char* out, int cap) {
    const Peptide& p = ((DB*)h)->peptides[i];
    std::string s;
    char buf[64];
    auto fmt = [&](float m) { double d = m; if (d == std::floor(d)) snprintf(buf, sizeof buf, "%+.0f", d); else snprintf(buf, sizeof buf, "%+g", d); return std::string(buf); };
    if (p.nterm) s += "[" + fmt(*p.nterm) + "]-";
    for (size_t k = 0; k < p.sequence.size(); k++) {
        s += p.sequence[k];
        if (p.modifications[k] != 0.0f) s += "[" + fmt(p.modifications[k]) + "]";
    }
    if (p.cterm) s += "-[" + fmt(*p.cterm) + "]";
    snprintf(out, cap, "%s", s.c_str());
    return (int)p.proteins.size();
}
int so_db_peptide_protein(void* h, uint64_t i, uint64_t j, char* out, int cap) {
    const Peptide& p = ((DB*)h)->peptides[i];
    if (j >= p.proteins.size()) return -1;
    snprintf(out, cap, "%s", p.proteins[j].c_str());
    return 0;
}

static Scorer make_scorer(const DB* db, const so_scorer_params* sp) {
    Scorer s;
    s.db = db;
    s.precursor_tol = {sp->precursor_tol.kind, sp->precursor_tol.lo, sp->precursor_tol.hi};
    s.fragment_tol = {sp->fragment_tol.kind, sp->fragment_tol.lo, sp->fragment_tol.hi};
    s.min_matched_peaks = sp->min_matched_peaks; s.min_isotope_err = sp->min_isotope_err; s.max_isotope_err = sp->max_isotope_err;
    s.min_precursor_charge = sp->min_precursor_charge; s.max_precursor_charge = sp->max_precursor_charge;
    s.override_precursor_charge = sp->override_precursor_charge; s.max_fragment_charge = sp->max_fragment_charge;
    s.chimera = sp->chimera; s.report_psms = sp->report_psms; s.wide_window = sp->wide_window;
    s.annotate_matches = sp->annotate_matches; s.score_type = sp->score_type;
    return s;
}

// Score a batch of spectra (SoA). Returns 0, or -(i+1)*4-{1,2} style error = reference panic on spectrum i.
// out must hold n*report_psms features; out_counts[i] = number of features of spectrum i (stored at out[i*report_psms ..]).
int64_t so_score_batch(void* h, const so_scorer_params* sp, uint64_t n, const uint64_t* peak_off, const float* masses, const float* intens,
                       const float* prec_mz, const uint8_t* prec_charge /*0=None*/, const float* iso_lo /*NaN=None*/, const float* iso_hi,
                       const float* tic, const uint8_t* level /*nullable: all 2*/, const float* ims /*nullable*/, int nthreads,
                       so_feature* out, uint32_t* out_counts, so_fragment* frag_out, uint64_t frag_cap, uint64_t* frag_used, so_counters* ctr_out) {
    DB* db = (DB*)h;
    Scorer sc = make_scorer(db, sp);
    int64_t err = 0;
    Counters total;
    std::vector<std::vector<Feature>> annotated(sp->annotate_matches ? n : 0);
#ifdef _OPENMP
    if (nthreads > 0) omp_set_num_threads(nthreads);
#endif
#pragma omp parallel
    {
        Counters local;
#pragma omp for schedule(dynamic, 16)
        for (int64_t i = 0; i < (int64_t)n; i++) {
            Spectrum q;
            q.level = level ? level[i] : 2;
            q.has_precursor = !std::isnan(prec_mz[i]);
            q.precursor.mz = prec_mz[i];
            if (prec_charge[i]) q.precursor.charge = prec_charge[i];
            if (!std::isnan(iso_lo[i]) && !std::isnan(iso_hi[i])) q.precursor.isolation_window = Tolerance{DA, iso_lo[i], iso_hi[i]};
            if (ims && !std::isnan(ims[i])) q.precursor.inverse_ion_mobility = ims[i];
            q.masses = masses + peak_off[i]; q.intensities = intens + peak_off[i]; q.n_peaks = (size_t)(peak_off[i + 1] - peak_off[i]);
            q.total_ion_current = tic[i];
            std::vector<Feature> feats;
            int rc = sc.score(q, feats, ctr_out ? &local : nullptr);
            if (rc != 0) {
#pragma omp critical
                { if (err == 0) err = -((int64_t)i * 4 + (-rc)); }
                out_counts[i] = 0;
                continue;
            }
            out_counts[i] = (uint32_t)feats.size();
            for (size_t r = 0; r < feats.size(); r++) {
                const Feature& f = feats[r];
                so_feature& o = out[(size_t)i * sp->report_psms + r];
                o.spectrum = (uint32_t)i; o.peptide_idx = f.peptide_idx; o.peptide_len = f.peptide_len; o.rank = f.rank; o.label = f.label;
                o.expmass = f.expmass; o.calcmass = f.calcmass; o.charge = f.charge; o.delta_mass = f.delta_mass; o.isotope_error = f.isotope_error;
                o.average_ppm = f.average_ppm; o.hyperscore = f.hyperscore; o.delta_next = f.delta_next; o.delta_best = f.delta_best;
                o.matched_peaks = f.matched_peaks; o.longest_b = f.longest_b; o.longest_y = f.longest_y; o.longest_y_pct = f.longest_y_pct;
                o.missed_cleavages = f.missed_cleavages; o.matched_intensity_pct = f.matched_intensity_pct; o.scored_candidates = f.scored_candidates;
                o.poisson = f.poisson; o.ms2_intensity = f.ms2_intensity; o.frag_offset = 0; o.frag_count = 0;
            }
            if (sp->annotate_matches) annotated[(size_t)i] = std::move(feats);
        }
#pragma omp critical
        total.add(local);
    }
    if (sp->annotate_matches && frag_out) {
        uint64_t used = 0;
        for (uint64_t i = 0; i < n; i++)
            for (size_t r = 0; r < annotated[i].size(); r++) {
                const Fragments& fr = annotated[i][r].fragments;
                so_feature& o = out[i * sp->report_psms + r];
                o.frag_offset = (uint32_t)used; o.frag_count = (uint32_t)fr.kinds.size();
                for (size_t k = 0; k < fr.kinds.size(); k++) {
                    if (used < frag_cap) frag_out[used] = {fr.kinds[k], fr.charges[k], fr.fragment_ordinals[k], fr.intensities[k], fr.mz_calculated[k], fr.mz_experimental[k]};
                    used++;
                }
            }
        if (frag_used) *frag_used = used;
    }
    if (ctr_out) {
        *ctr_out = {total.queries, total.probes_pep, total.probes_bucket, total.pages, total.probes_page, total.entries_scanned,
                    total.candidates_scored, total.psms, total.peptide_record_floats};
    }
    return err;
}

// Scorer::quick_score over a batch; keep[n_peptides] bytes are OR-ed (AtomicBool store(true)).
int64_t so_quick_score(void* h, const so_scorer_params* sp, uint64_t n, const uint64_t* peak_off, const float* masses, const float* intens,
                       const float* prec_mz, const uint8_t* prec_charge, const float* iso_lo, const float* iso_hi, const float* tic, int low_memory,
                       uint8_t* keep) {
    DB* db = (DB*)h;
    Scorer sc = make_scorer(db, sp);
    for (uint64_t i = 0; i < n; i++) {
        Spectrum q;
        q.has_precursor = !std::isnan(prec_mz[i]);
        q.precursor.mz = prec_mz[i];
        if (prec_charge[i]) q.precursor.charge = prec_charge[i];
        if (!std::isnan(iso_lo[i]) && !std::isnan(iso_hi[i])) q.precursor.isolation_window = Tolerance{DA, iso_lo[i], iso_hi[i]};
        q.masses = masses + peak_off[i]; q.intensities = intens + peak_off[i]; q.n_peaks = (size_t)(peak_off[i + 1] - peak_off[i]);
        q.total_ion_current = tic[i];
        int rc = sc.quick_score(q, low_memory != 0, keep);
        if (rc) return -((int64_t)i * 4 + (-rc));
    }
    return 0;
}

// Preliminary hits of one spectrum (after initial_hits), in heap order, for white-box parity of the trim kernels.
int64_t so_initial_hits(void* h, const so_scorer_params* sp, const float* masses, const float* intens, uint64_t n_peaks, float prec_mz,
                        uint8_t prec_charge, float iso_lo, float iso_hi, uint16_t* matched, uint32_t* peptide, uint8_t* charge, int8_t* iso,
                        uint64_t cap, uint64_t* matched_peaks, uint64_t* scored_candidates) {
    Scorer sc = make_scorer((DB*)h, sp);
    Spectrum q; q.masses = masses; q.intensities = intens; q.n_peaks = (size_t)n_peaks; q.precursor.mz = prec_mz;
    if (prec_charge) q.precursor.charge = prec_charge;
    if (!std::isnan(iso_lo) && !std::isnan(iso_hi)) q.precursor.isolation_window = Tolerance{DA, iso_lo, iso_hi};
    InitialHits hits = sc.initial_hits(q, q.precursor, nullptr);
    *matched_peaks = hits.matched_peaks; *scored_candidates = hits.scored_candidates;
    for (size_t i = 0; i < hits.preliminary.size() && i < cap; i++) {
        matched[i] = hits.preliminary[i].matched; peptide[i] = hits.preliminary[i].peptide;
        charge[i] = hits.preliminary[i].precursor_charge; iso[i] = hits.preliminary[i].isotope_error;
    }
    return (int64_t)hits.preliminary.size();
}

// ---- unit-level entry points for the ported reference known-answer tests
void so_tolerance_bounds(int kind, float lo, float hi, float center, float* out) { Tolerance{kind, lo, hi}.bounds(center, out[0], out[1]); }
void so_binary_search_slice_f64(const double* data, uint64_t n, double low, double high, uint64_t* out) {
    size_t l, r;
    binary_search_slice((size_t)n, [&](size_t k) { return f64_key(data[k]) < f64_key(low); }, [&](size_t k) { return f64_key(data[k]) <= f64_key(high); }, l, r);
    out[0] = l; out[1] = r;
}
void so_binary_search_slice_f32(const float* data, uint64_t n, float low, float high, uint64_t* out) {
    size_t l, r;
    binary_search_slice((size_t)n, [&](size_t k) { return total_cmp(data[k], low) < 0; }, [&](size_t k) { return total_cmp(data[k], high) <= 0; }, l, r);
    out[0] = l; out[1] = r;
}
uint8_t so_max_fragment_charge(int opt, uint8_t z) { return so::max_fragment_charge(opt, z); }
void so_bounded_min_heapify_i32(int32_t* data, uint64_t n, uint64_t k) { bounded_min_heapify(data, (size_t)n, (size_t)k, [](int32_t a, int32_t b) { return a < b; }); }
void so_bounded_min_heapify_u64(uint64_t* data, uint64_t n, uint64_t k) { bounded_min_heapify(data, (size_t)n, (size_t)k, [](uint64_t a, uint64_t b) { return a < b; }); }
void so_run(const uint64_t* idx, uint64_t n, uint64_t* out) {
    Run r;
    for (uint64_t i = 0; i < n; i++) r.matched((size_t)idx[i]);
    out[0] = r.start; out[1] = r.length; out[2] = r.last; out[3] = r.longest;
}
// ion series of a bare peptide (Peptide::try_from(Digest)) with optional per-residue mods / nterm / cterm added to monoisotopic
uint64_t so_ion_series(const char* seq, const float* mods /*nullable*/, float nterm /*NaN none*/, float cterm, int kind, float* out, float* mono_out) {
    Digest d; d.sequence = seq;
    Peptide p;
    if (!peptide_from_digest(d, p)) return 0;
    if (mods) for (size_t i = 0; i < p.modifications.size(); i++) p.modifications[i] = mods[i];
    if (!std::isnan(nterm)) p.nterm = nterm;
    if (!std::isnan(cterm)) p.cterm = cterm;
    p.monoisotopic += modification_mass(p);
    std::vector<float> ions;
    ion_series(p, kind, ions);
    for (size_t i = 0; i < ions.size(); i++) out[i] = ions[i];
    if (mono_out) *mono_out = p.monoisotopic;
    return ions.size();
}
int so_select_most_intense_peak(const float* masses, const float* intens, uint64_t n, float center, int kind, float lo, float hi, float offset /*NaN none*/) {
    return select_most_intense_peak(masses, intens, (size_t)n, center, Tolerance{kind, lo, hi}, std::isnan(offset) ? std::nullopt : std::optional<float>(offset));
}
void so_deisotope(const float* mz, const float* inten, uint64_t n, uint8_t max_charge, float ppm, float min_mz, int compress, float* out_int, int32_t* out_charge,
                  int64_t* out_env) {
    auto d = deisotope(mz, inten, (size_t)n, max_charge, ppm, min_mz);
    if (compress) path_compression(d);
    for (size_t i = 0; i < d.size(); i++) { out_int[i] = d[i].intensity; out_charge[i] = d[i].charge; out_env[i] = d[i].envelope; }
}
uint64_t so_process_ms2(const float* mz, const float* inten, uint64_t n, int precursor_charge, uint64_t take_top_n, int do_deisotope, float min_deisotope_mz,
                        float* out_mass, float* out_int, float* out_tic) {
    std::vector<float> m, i;
    float tic;
    process_ms2(mz, inten, (size_t)n, precursor_charge, (size_t)take_top_n, do_deisotope, min_deisotope_mz, m, i, tic);
    std::memcpy(out_mass, m.data(), 4 * m.size());
    std::memcpy(out_int, i.data(), 4 * i.size());
    *out_tic = tic;
    return m.size();
}
// db.query(precursor_mass, ptol, ftol).page_search(mass) -> visited fragments (crates/sage/tests/integration.rs:30-70)
uint64_t so_page_search(void* h, float precursor_mass, so_tol ptol, so_tol ftol, float mass, uint32_t* out_pep, float* out_mz, uint64_t cap, uint64_t* pre_lo_hi) {
    DB* db = (DB*)h;
    IndexedQuery q = db_query(*db, precursor_mass, Tolerance{ptol.kind, ptol.lo, ptol.hi}, Tolerance{ftol.kind, ftol.lo, ftol.hi}, nullptr);
    if (pre_lo_hi) { pre_lo_hi[0] = q.pre_idx_lo; pre_lo_hi[1] = q.pre_idx_hi; }
    uint64_t n = 0;
    page_search(q, mass, nullptr, [&](const Theoretical& f) { if (n < cap) { out_pep[n] = f.peptide_index; out_mz[n] = f.fragment_mz; } n++; });
    return n;
}
// tmt.rs:193-211 find_reporter_ions (+ unwrap_or_default of tmt.rs:333): intensity of the most intense peak within tolerance of each label, else 0
void so_find_reporter_ions(uint64_t n, const uint64_t* peak_off, const float* masses, const float* intens, const float* labels, uint64_t n_labels, so_tol tol,
                           float* out) {
    for (uint64_t i = 0; i < n; i++)
        for (uint64_t l = 0; l < n_labels; l++) {
            const int pk = select_most_intense_peak(masses + peak_off[i], intens + peak_off[i], (size_t)(peak_off[i + 1] - peak_off[i]), labels[l],
                                                    Tolerance{tol.kind, tol.lo, tol.hi}, std::optional<float>(-PROTON));
            out[i * n_labels + l] = pk >= 0 ? intens[peak_off[i] + pk] : 0.0f;
        }
}
// Score::hyperscore (scoring.rs:179-201) and the ln-factorial approximation (:170-177) on their own, for the high-precision cross-check in
// tests/test_oracle_known_answers.py (the f64 fields are otherwise pinned only by the oracle itself).
double so_hyperscore(int32_t score_type, uint32_t matched_b, uint32_t matched_y, float summed_b, float summed_y) {
    return score_type_score(score_type, (uint16_t)matched_b, (uint16_t)matched_y, summed_b, summed_y);
}
double so_lnfact(uint32_t n) { return lnfact((uint16_t)n); }
int so_num_threads() {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

}  // extern "C"
