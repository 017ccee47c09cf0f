// CPU oracle of MgfReader::parse (sage-cloudpath mgf.rs:324-370, util.rs:107-118), written line by line from the Rust, single-threaded
// like the reference reader. Numbers: the token is checked against the grammar of Rust's f32::from_str, then converted by glibc strtof
// (correctly rounded in the C locale); inf / infinity / nan are spelled out. The sum is a left fold from +0.0 compiled without contraction,
// so each step is one SSE addss with x86's NaN rules; RTINSECONDS / 60.0 is one divss.
#include <clocale>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

namespace {

bool is_digit(unsigned char c) { return c >= '0' && c <= '9'; }

// Rust's dec2flt grammar, then the value.
bool parse_f32(const std::string& s, float* out) {
    size_t i = 0, n = s.size();
    if (n == 0) return false;
    bool neg = s[0] == '-';
    if (s[0] == '-' || s[0] == '+') i++;
    if (i == n) return false;
    std::string rest = s.substr(i);
    std::string low;
    for (char c : rest) low += (char)((c >= 'A' && c <= 'Z') ? c + 32 : c);
    if (low == "inf" || low == "infinity") { *out = neg ? -INFINITY : INFINITY; return true; }
    if (low == "nan") { uint32_t u = neg ? 0xFFC00000u : 0x7FC00000u; memcpy(out, &u, 4); return true; }
    size_t nd = 0;
    while (i < n && is_digit(s[i])) { i++; nd++; }
    if (i < n && s[i] == '.') { i++; while (i < n && is_digit(s[i])) { i++; nd++; } }
    if (nd == 0) return false;
    if (i < n && (s[i] == 'e' || s[i] == 'E')) {
        i++;
        if (i < n && (s[i] == '+' || s[i] == '-')) i++;
        if (i == n || !is_digit(s[i])) return false;
        while (i < n && is_digit(s[i])) i++;
    }
    if (i != n) return false;
    *out = strtof(s.c_str(), nullptr);
    return true;
}

// char::is_whitespace (Unicode White_Space), decoded from valid UTF-8
size_t ws_front(const std::string& s, size_t b, size_t e) {
    const unsigned char* t = (const unsigned char*)s.data();
    unsigned char c = t[b];
    if (c == ' ' || (c >= 0x09 && c <= 0x0D)) return 1;
    if (e - b >= 2 && c == 0xC2 && (t[b + 1] == 0x85 || t[b + 1] == 0xA0)) return 2;
    if (e - b >= 3 && c >= 0xE0 && c < 0xF0) {
        uint32_t cp = ((c & 0x0F) << 12) | ((t[b + 1] & 0x3F) << 6) | (t[b + 2] & 0x3F);
        if (cp == 0x1680 || (cp >= 0x2000 && cp <= 0x200A) || cp == 0x2028 || cp == 0x2029 || cp == 0x202F || cp == 0x205F || cp == 0x3000) return 3;
    }
    return 0;
}
size_t ws_back(const std::string& s, size_t b, size_t e) {
    const unsigned char* t = (const unsigned char*)s.data();
    unsigned char c = t[e - 1];
    if (c == ' ' || (c >= 0x09 && c <= 0x0D)) return 1;
    if (e - b >= 2 && t[e - 2] == 0xC2 && (c == 0x85 || c == 0xA0)) return 2;
    if (e - b >= 3 && t[e - 3] >= 0xE0 && t[e - 3] < 0xF0) {
        uint32_t cp = ((t[e - 3] & 0x0F) << 12) | ((t[e - 2] & 0x3F) << 6) | (c & 0x3F);
        if (cp == 0x1680 || (cp >= 0x2000 && cp <= 0x200A) || cp == 0x2028 || cp == 0x2029 || cp == 0x202F || cp == 0x205F || cp == 0x3000) return 3;
    }
    return 0;
}
std::string trim(const std::string& s, size_t b, size_t e) {
    while (b < e) { size_t k = ws_front(s, b, e); if (!k) break; b += k; }
    while (b < e) { size_t k = ws_back(s, b, e); if (!k) break; e -= k; }
    return s.substr(b, e - b);
}

// the first invalid offset of a UTF-8 string, or -1
int64_t utf8_error(const unsigned char* t, size_t n) {
    size_t i = 0;
    while (i < n) {
        unsigned char c = t[i];
        size_t len = c < 0x80 ? 1 : c < 0xC2 ? 0 : c < 0xE0 ? 2 : c < 0xF0 ? 3 : c < 0xF5 ? 4 : 0;
        if (len == 0 || i + len > n) return (int64_t)i;
        for (size_t k = 1; k < len; k++)
            if ((t[i + k] & 0xC0) != 0x80) return (int64_t)i;
        if ((c == 0xE0 && t[i + 1] < 0xA0) || (c == 0xED && t[i + 1] > 0x9F) || (c == 0xF0 && t[i + 1] < 0x90) || (c == 0xF4 && t[i + 1] > 0x8F))
            return (int64_t)i;
        i += len;
    }
    return -1;
}

bool starts_with(const std::string& s, const char* p) { return s.compare(0, strlen(p), p) == 0; }
bool strip_prefix(const std::string& s, const char* p, std::string& rest) {
    if (!starts_with(s, p)) return false;
    rest = s.substr(strlen(p));
    return true;
}
bool ascii_ws(char c) { return c == ' ' || c == '\t' || c == '\n' || c == '\x0C' || c == '\r'; }
std::vector<std::string> split_ascii_whitespace(const std::string& s) {
    std::vector<std::string> out;
    size_t i = 0;
    while (i < s.size()) {
        while (i < s.size() && ascii_ws(s[i])) i++;
        if (i == s.size()) break;
        size_t b = i;
        while (i < s.size() && !ascii_ws(s[i])) i++;
        out.push_back(s.substr(b, i - b));
    }
    return out;
}
// regex (\d)\+? over the string, each match's first char .to_digit(10): the ASCII digits in order
std::vector<uint8_t> charges(const std::string& s) {
    std::vector<uint8_t> v;
    for (char c : s)
        if (is_digit(c)) v.push_back((uint8_t)(c - '0'));
    return v;
}

struct Precursor { float mz = 0.0f; bool int_some = false; float intensity = 0.0f; bool charge_some = false; uint8_t charge = 0;
                   uint8_t iso = 0; float lo = 0.0f, hi = 0.0f; };
struct Spectrum { std::string id; float rt = 0.0f, tic = 0.0f; std::vector<Precursor> precursors; std::vector<float> mz, intensity; };

template <class T>
struct Opt { bool some = false; T v{}; void set(const T& x) { some = true; v = x; } };

struct Result {
    int rc = 0;
    std::string error;
    uint64_t n_lines = 0, n_records = 0, malformed = 0;
    std::vector<Spectrum> spectra;
};

void parse(const char* text, size_t len, Result& R) {
    int64_t bad = utf8_error((const unsigned char*)text, len);
    if (bad >= 0) { R.rc = -1; R.error = "invalid UTF-8 at byte offset " + std::to_string(bad); return; }
    std::string s(text, len);
    // str::lines
    std::vector<std::string> lines;
    size_t b = 0;
    while (b < len) {
        size_t e = s.find('\n', b);
        if (e == std::string::npos) { lines.push_back(s.substr(b)); break; }
        lines.push_back(s.substr(b, e - b));
        b = e + 1;
    }
    R.n_lines = lines.size();
    size_t li = 0;
    // header (DefaultParser): begin, tol, tolu, charge
    Opt<float> d_tol;
    Opt<std::string> d_tolu;
    Opt<std::vector<uint8_t>> d_charge;
    bool started = false;
    while (!started) {
        if (li == lines.size()) { R.rc = -1; R.error = "no BEGIN IONS line"; return; }
        std::string line = trim(lines[li], 0, lines[li].size());
        li++;
        std::string rest;
        if (starts_with(line, "BEGIN IONS")) started = true;
        else if (strip_prefix(line, "TOL=", rest)) { float v; if (parse_f32(rest, &v)) d_tol.set(v); }
        else if (strip_prefix(line, "TOLU=", rest)) d_tolu.set(rest);
        else if (strip_prefix(line, "CHARGE=", rest)) d_charge.set(charges(rest));
    }
    // QueryData::default_with_params: the first record starts from None
    std::string id;
    std::vector<Precursor> precursors;
    Opt<float> tol, rt;
    Opt<std::string> tolu;
    Opt<std::vector<uint8_t>> charge;
    std::vector<float> mz, intensity;
    for (; li < lines.size(); li++) {
        std::string line = trim(lines[li], 0, lines[li].size());
        std::string rest;
        if (!line.empty() && is_digit(line[0])) {   // parse_mz (a non-ASCII numeric first char never parses)
            auto tok = split_ascii_whitespace(line);
            float v;
            if (!parse_f32(tok[0], &v)) { R.malformed++; continue; }
            mz.push_back(v);
            if (tok.size() >= 2) { if (parse_f32(tok[1], &v)) intensity.push_back(v); }
            else intensity.push_back(1.0f);
        } else if (starts_with(line, "END IONS")) {
            Spectrum sp;
            sp.id = id;
            uint8_t iso = 0;
            float lo = 0.0f, hi = 0.0f;
            if (tol.some && tolu.some && (tolu.v == "Da" || tolu.v == "ppm")) {
                iso = tolu.v == "Da" ? 1 : 2;
                hi = std::fabs(tol.v);
                lo = -hi;
            }
            for (Precursor p : precursors) {
                p.iso = iso; p.lo = lo; p.hi = hi;
                if (charge.some) {
                    for (uint8_t c : charge.v) { Precursor q = p; q.charge_some = true; q.charge = c; sp.precursors.push_back(q); }
                } else sp.precursors.push_back(p);
            }
            sp.rt = rt.some ? rt.v : 0.0f;
            float t = 0.0f;
            for (float x : intensity) t = t + x;
            sp.tic = t;
            sp.mz = mz;
            sp.intensity = intensity;
            R.n_records++;
            if (!(sp.id.empty() || sp.precursors.empty() || sp.mz.empty() || sp.mz.size() != sp.intensity.size())) R.spectra.push_back(sp);
            // init()
            id.clear(); precursors.clear(); tol = d_tol; tolu = d_tolu; charge = d_charge; rt = Opt<float>(); mz.clear(); intensity.clear();
        } else if (strip_prefix(line, "PEPMASS=", rest)) {
            auto tok = split_ascii_whitespace(rest);
            Precursor p;
            float v;
            if (!tok.empty()) {
                if (!parse_f32(tok[0], &v)) { R.malformed++; continue; }
                p.mz = v;
            }
            if (tok.size() >= 2 && parse_f32(tok[1], &v)) { p.int_some = true; p.intensity = v; }
            precursors.push_back(p);
        } else if (strip_prefix(line, "TITLE=", rest)) {
            id = rest;
        } else if (strip_prefix(line, "CHARGE=", rest)) {
            charge.set(charges(rest));
        } else if (strip_prefix(line, "TOL=", rest)) {
            float v;
            if (parse_f32(rest, &v)) tol.set(v);
        } else if (strip_prefix(line, "TOLU=", rest)) {
            tolu.set(rest);
        } else if (strip_prefix(line, "RTINSECONDS=", rest)) {
            float v;
            if (parse_f32(rest, &v)) rt.set(v / 60.0f);
        }
    }
}

}  // namespace

extern "C" {

void* mo_create(const char* text, uint64_t len) {
    setlocale(LC_NUMERIC, "C");
    Result* R = new Result();
    parse(text, len, *R);
    return R;
}
void mo_destroy(void* h) { delete (Result*)h; }
// rc, then n_lines, n_records, n_spectra, n_peaks, n_precursors, id_bytes, malformed
int mo_info(void* h, uint64_t* out, char* err, uint64_t cap) {
    Result* R = (Result*)h;
    uint64_t npk = 0, npr = 0, nid = 0;
    for (auto& s : R->spectra) { npk += s.mz.size(); npr += s.precursors.size(); nid += s.id.size(); }
    const uint64_t v[7] = {R->n_lines, R->n_records, (uint64_t)R->spectra.size(), npk, npr, nid, R->malformed};
    memcpy(out, v, sizeof v);
    if (err && cap) { strncpy(err, R->error.c_str(), cap - 1); err[cap - 1] = 0; }
    return R->rc;
}
void mo_export(void* h, uint64_t* peak_off, float* mz, float* intensity, float* rt, float* tic, uint64_t* prec_off, float* p_mz, float* p_int,
               uint8_t* p_int_some, uint8_t* p_charge, uint8_t* p_charge_some, uint8_t* p_iso, float* p_lo, float* p_hi, uint64_t* id_off, char* id) {
    Result* R = (Result*)h;
    uint64_t a = 0, b = 0, c = 0, k = 0;
    peak_off[0] = prec_off[0] = id_off[0] = 0;
    for (auto& s : R->spectra) {
        for (size_t i = 0; i < s.mz.size(); i++, a++) { mz[a] = s.mz[i]; intensity[a] = s.intensity[i]; }
        for (auto& p : s.precursors) {
            p_mz[b] = p.mz; p_int[b] = p.intensity; p_int_some[b] = p.int_some; p_charge[b] = p.charge; p_charge_some[b] = p.charge_some;
            p_iso[b] = p.iso; p_lo[b] = p.lo; p_hi[b] = p.hi; b++;
        }
        memcpy(id + c, s.id.data(), s.id.size());
        c += s.id.size();
        rt[k] = s.rt;
        tic[k] = s.tic;
        k++;
        peak_off[k] = a; prec_off[k] = b; id_off[k] = c;
    }
}
// str::parse::<f32> of each token
void mo_parse_f32(const char* bytes, const uint64_t* off, uint64_t n, float* out, uint8_t* ok) {
    setlocale(LC_NUMERIC, "C");
    for (uint64_t i = 0; i < n; i++) {
        float v = 0.0f;
        ok[i] = parse_f32(std::string(bytes + off[i], off[i + 1] - off[i]), &v);
        out[i] = ok[i] ? v : 0.0f;
    }
}

}
