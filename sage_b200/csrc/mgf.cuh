// MgfReader::parse (sage-cloudpath mgf.rs:324-370) on the device: the whole file's bytes are resident; positions and peak offsets are u64.
//
//   k_mgf_bytes       one thread per byte: UTF-8 validity (the first bad offset by atomicMin) and the count of '\n'
//                     (the host then lists the '\n' positions with cub::DeviceSelect)
//   k_mgf_lines       one thread per line (`str::lines`): Unicode `trim` of both ends, the line's kind from its prefix, and its numbers
//                     parsed in place (mgf_f32.cuh); the first BEGIN IONS line by atomicMin
//   k_mgf_scan_lines  one thread per line: header lines (up to the first BEGIN) give the file defaults (last TOL= that parses, last TOLU=,
//                     last CHARGE=) by atomicMax; later lines count malformed PEPMASS / peak lines and END IONS lines
//                     (the host lists the END lines with cub::DeviceSelect: record r ends at the r-th one)
//   k_mgf_records     one thread per record, in file order over its lines: the last-wins fields, the defaults from record 1 on, the
//                     counts and the drop check (pass 0); then, at the places cub's scans gave, the spectrum's arrays and id (pass 1).
//                     The TIC is the serial f32 sum in file order (tic_add: x86's NaN rules, from +0.0).
#pragma once
#include <stdint.h>

#include "mgf_f32.cuh"
#include "spectra.cuh"   // tic_add, raw_quiet

namespace sb {

enum MgfKind : uint8_t { MGF_OTHER = 0, MGF_BEGIN, MGF_END, MGF_PEAK, MGF_PEPMASS, MGF_TITLE, MGF_CHARGE, MGF_TOL, MGF_TOLU, MGF_RT };
enum MgfUnit : uint8_t { MGF_UNIT_OTHER = 0, MGF_UNIT_DA = 1, MGF_UNIT_PPM = 2 };

// One line after trim. beg/end: the value after the prefix (TITLE, TOLU, CHARGE) or the trimmed line. a/b and fa/fb by kind:
//   PEAK     a = m/z, fa = it parsed; b = intensity, fb = 0 no second token (1.0 is pushed) / 1 parsed / 2 failed
//   PEPMASS  a = m/z, fa = 0 no token (0.0) / 1 parsed / 2 failed; b = intensity, fb = it parsed (Some)
//   TOL, RT  a = value, fa = it parsed;     TOLU  fa = MgfUnit;     CHARGE  count = its ASCII digits
struct MgfLine {
    uint64_t beg, end, count;
    float a, b;
    uint8_t kind, fa, fb;
};

struct MgfHeader {
    unsigned long long begin_line;            // first BEGIN IONS line, ~0 if none
    unsigned long long tol, tolu, charge;     // 1 + the header line that sets the default, 0 = None
    unsigned long long malformed, n_end;      // after the header
    unsigned long long bad_utf8, n_newline;   // first invalid byte offset (~0: valid), '\n' count
};

// ---------------------------------------------------------------------------------------------------------------------------------- UTF-8
// A byte is bad when it leads an invalid sequence (Rust's from_utf8 rules: no overlong forms, no surrogates, <= U+10FFFF, complete), or
// is a continuation byte no lead byte of the three before covers. The smallest bad offset is from_utf8's valid_up_to.
__device__ __forceinline__ bool mgf_cont(uint8_t c) { return (c & 0xC0) == 0x80; }
__device__ __forceinline__ int mgf_seq_len(uint8_t c) { return c < 0x80 ? 1 : c < 0xC2 ? 0 : c < 0xE0 ? 2 : c < 0xF0 ? 3 : c < 0xF5 ? 4 : 0; }

__device__ inline bool mgf_byte_bad(const uint8_t* t, uint64_t n, uint64_t i) {
    const uint8_t c = t[i];
    if (c < 0x80) return false;
    if (mgf_cont(c)) {
        for (int back = 1; back <= 3 && back <= (int)i; back++) {
            const uint8_t l = t[i - back];
            if (mgf_cont(l)) continue;
            return mgf_seq_len(l) <= back;   // a lead byte this far back must reach i (its own validity is its own check)
        }
        return true;
    }
    const int len = mgf_seq_len(c);
    if (len == 0 || i + len > n) return true;
    for (int k = 1; k < len; k++)
        if (!mgf_cont(t[i + k])) return true;
    const uint8_t c1 = t[i + 1];
    if (c == 0xE0 && c1 < 0xA0) return true;   // overlong
    if (c == 0xED && c1 > 0x9F) return true;   // surrogates
    if (c == 0xF0 && c1 < 0x90) return true;   // overlong
    if (c == 0xF4 && c1 > 0x8F) return true;   // > U+10FFFF
    return false;
}

__global__ void k_mgf_bytes(const uint8_t* t, uint64_t n, MgfHeader* h) {
    unsigned long long bad = ~0ull, nl = 0;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        if (t[i] == '\n') nl++;
        if (bad == ~0ull && mgf_byte_bad(t, n, i)) bad = i;
    }
    for (int o = 16; o; o >>= 1) {
        nl += __shfl_xor_sync(0xffffffffu, nl, o);
        bad = min(bad, __shfl_xor_sync(0xffffffffu, bad, o));
    }
    if ((threadIdx.x & 31) == 0) {
        if (nl) atomicAdd(&h->n_newline, nl);
        if (bad != ~0ull) atomicMin(&h->bad_utf8, bad);
    }
}

// ---------------------------------------------------------------------------------------------------------------------------------- lines
// Unicode White_Space (char::is_whitespace, what str::trim strips) ending at t[e - 1] / starting at t[b]: its byte length, 0 if none.
__device__ inline int mgf_ws_back(const uint8_t* t, uint64_t b, uint64_t e) {
    const uint64_t n = e - b;
    const uint8_t c = t[e - 1];
    if (c == ' ' || (c >= 0x09 && c <= 0x0D)) return 1;
    if (n >= 2 && t[e - 2] == 0xC2 && (c == 0x85 || c == 0xA0)) return 2;
    if (n >= 3) {
        const uint8_t x = t[e - 3], y = t[e - 2];
        if (x == 0xE1 && y == 0x9A && c == 0x80) return 3;                                                      // U+1680
        if (x == 0xE2 && y == 0x80 && ((c >= 0x80 && c <= 0x8A) || c == 0xA8 || c == 0xA9 || c == 0xAF)) return 3;   // U+2000-200A, 2028/9, 202F
        if (x == 0xE2 && y == 0x81 && c == 0x9F) return 3;                                                      // U+205F
        if (x == 0xE3 && y == 0x80 && c == 0x80) return 3;                                                      // U+3000
    }
    return 0;
}
__device__ inline int mgf_ws_front(const uint8_t* t, uint64_t b, uint64_t e) {
    const uint64_t n = e - b;
    const uint8_t c = t[b];
    if (c == ' ' || (c >= 0x09 && c <= 0x0D)) return 1;
    if (n >= 2 && c == 0xC2 && (t[b + 1] == 0x85 || t[b + 1] == 0xA0)) return 2;
    if (n >= 3) {
        const uint8_t y = t[b + 1], z = t[b + 2];
        if (c == 0xE1 && y == 0x9A && z == 0x80) return 3;
        if (c == 0xE2 && y == 0x80 && ((z >= 0x80 && z <= 0x8A) || z == 0xA8 || z == 0xA9 || z == 0xAF)) return 3;
        if (c == 0xE2 && y == 0x81 && z == 0x9F) return 3;
        if (c == 0xE3 && y == 0x80 && z == 0x80) return 3;
    }
    return 0;
}

// u8::is_ascii_whitespace, what split_ascii_whitespace splits at (no vertical tab)
__device__ __forceinline__ bool mgf_ascii_ws(uint8_t c) { return c == ' ' || c == '\t' || c == '\n' || c == '\x0C' || c == '\r'; }

__device__ inline bool mgf_prefix(const uint8_t* t, uint64_t b, uint64_t e, const char* p, uint64_t& rest) {
    uint64_t i = 0;
    for (; p[i]; i++)
        if (b + i >= e || t[b + i] != (uint8_t)p[i]) return false;
    rest = b + i;
    return true;
}

// The next split_ascii_whitespace token of [*p, e): [tb, te); false when none is left.
__device__ inline bool mgf_token(const uint8_t* t, uint64_t& p, uint64_t e, uint64_t& tb, uint64_t& te) {
    while (p < e && mgf_ascii_ws(t[p])) p++;
    if (p == e) return false;
    tb = p;
    while (p < e && !mgf_ascii_ws(t[p])) p++;
    te = p;
    return true;
}

__device__ __forceinline__ bool mgf_num(const uint8_t* t, uint64_t b, uint64_t e, float& v) { return mgf_parse_f32(t + b, e - b, &v); }

__global__ void k_mgf_lines(const uint8_t* t, uint64_t n, const uint64_t* nl, uint64_t n_nl, uint64_t n_lines, MgfLine* L, MgfHeader* h) {
    for (uint64_t l = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; l < n_lines; l += (uint64_t)gridDim.x * blockDim.x) {
        uint64_t b = l == 0 ? 0 : nl[l - 1] + 1, e = l < n_nl ? nl[l] : n;
        while (b < e) { const int k = mgf_ws_front(t, b, e); if (!k) break; b += k; }
        while (b < e) { const int k = mgf_ws_back(t, b, e); if (!k) break; e -= k; }
        MgfLine o{b, e, 0, 0.0f, 0.0f, MGF_OTHER, 0, 0};
        uint64_t r = 0;
        if (b < e && t[b] >= '0' && t[b] <= '9') {
            o.kind = MGF_PEAK;
            uint64_t p = b, tb, te;
            mgf_token(t, p, e, tb, te);
            o.fa = mgf_num(t, tb, te, o.a);
            if (mgf_token(t, p, e, tb, te)) o.fb = mgf_num(t, tb, te, o.b) ? 1 : 2;
        } else if (mgf_prefix(t, b, e, "END IONS", r)) {
            o.kind = MGF_END;
        } else if (mgf_prefix(t, b, e, "PEPMASS=", r)) {
            o.kind = MGF_PEPMASS;
            uint64_t p = r, tb, te;
            if (mgf_token(t, p, e, tb, te)) {
                o.fa = mgf_num(t, tb, te, o.a) ? 1 : 2;
                if (mgf_token(t, p, e, tb, te)) o.fb = mgf_num(t, tb, te, o.b);
            }
        } else if (mgf_prefix(t, b, e, "TITLE=", r)) {
            o.kind = MGF_TITLE;
            o.beg = r;
        } else if (mgf_prefix(t, b, e, "CHARGE=", r)) {
            o.kind = MGF_CHARGE;
            o.beg = r;
            for (uint64_t i = r; i < e; i++) o.count += t[i] >= '0' && t[i] <= '9';
        } else if (mgf_prefix(t, b, e, "TOL=", r)) {
            o.kind = MGF_TOL;
            o.fa = mgf_num(t, r, e, o.a);
        } else if (mgf_prefix(t, b, e, "TOLU=", r)) {
            o.kind = MGF_TOLU;
            o.beg = r;
            const uint64_t m = e - r;
            o.fa = (m == 2 && t[r] == 'D' && t[r + 1] == 'a') ? MGF_UNIT_DA : (m == 3 && t[r] == 'p' && t[r + 1] == 'p' && t[r + 2] == 'm') ? MGF_UNIT_PPM : MGF_UNIT_OTHER;
        } else if (mgf_prefix(t, b, e, "RTINSECONDS=", r)) {
            o.kind = MGF_RT;
            o.fa = mgf_num(t, r, e, o.a);
        } else if (mgf_prefix(t, b, e, "BEGIN IONS", r)) {
            o.kind = MGF_BEGIN;
            atomicMin(&h->begin_line, (unsigned long long)l);
        }
        L[l] = o;
    }
}

__global__ void k_mgf_scan_lines(const MgfLine* L, uint64_t n_lines, MgfHeader* h) {
    const uint64_t B = h->begin_line;
    unsigned long long bad = 0, ends = 0;
    for (uint64_t l = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; l < n_lines; l += (uint64_t)gridDim.x * blockDim.x) {
        const uint8_t k = L[l].kind;
        if (l <= B) {
            if (k == MGF_TOL && L[l].fa) atomicMax(&h->tol, (unsigned long long)l + 1);
            if (k == MGF_TOLU) atomicMax(&h->tolu, (unsigned long long)l + 1);
            if (k == MGF_CHARGE) atomicMax(&h->charge, (unsigned long long)l + 1);
        } else {
            bad += (k == MGF_PEAK && !L[l].fa) || (k == MGF_PEPMASS && L[l].fa == 2);
            ends += k == MGF_END;
        }
    }
    for (int o = 16; o; o >>= 1) {
        bad += __shfl_xor_sync(0xffffffffu, bad, o);
        ends += __shfl_xor_sync(0xffffffffu, ends, o);
    }
    if ((threadIdx.x & 31) == 0) {
        if (bad) atomicAdd(&h->malformed, bad);
        if (ends) atomicAdd(&h->n_end, ends);
    }
}

// ---------------------------------------------------------------------------------------------------------------------------------- records
struct MgfOut {
    // pass 0 writes each record's counts ([n_rec + 1], the last entry 0); pass 1 reads their exclusive scans (the record's places) here
    uint64_t *kept, *n_peaks, *n_prec, *id_len;
    // pass 1, indexed by kept spectrum k / peak / precursor / id byte
    uint64_t *peak_off, *prec_off, *id_off;
    float *mz, *intensity, *rt, *tic;
    float *p_mz, *p_int, *p_lo, *p_hi;
    uint8_t *p_int_some, *p_charge, *p_charge_some, *p_iso;
    uint8_t* id_bytes;
};

// Record r's state at END IONS (QueryData of mgf.rs), from its lines in file order.
struct MgfRecord {
    int64_t title, tol, tolu, charge, rt;   // the line that sets each field, -1 = None
    uint64_t n_pep, n_mz, n_int;
    float tic;
};

__device__ inline MgfRecord mgf_record(const MgfLine* L, uint64_t l0, uint64_t l1, bool first, const MgfHeader& h) {
    MgfRecord R{-1, -1, -1, -1, -1, 0, 0, 0, 0.0f};
    for (uint64_t l = l0; l < l1; l++) {
        const MgfLine& x = L[l];
        switch (x.kind) {
            case MGF_PEAK:
                if (x.fa) {
                    R.n_mz++;
                    if (x.fb != 2) {
                        R.n_int++;
                        R.tic = tic_add(R.tic, x.fb ? x.b : 1.0f);
                    }
                }
                break;
            case MGF_PEPMASS: R.n_pep += x.fa != 2; break;
            case MGF_TITLE: R.title = (int64_t)l; break;
            case MGF_CHARGE: R.charge = (int64_t)l; break;
            case MGF_TOL: if (x.fa) R.tol = (int64_t)l; break;
            case MGF_TOLU: R.tolu = (int64_t)l; break;
            case MGF_RT: if (x.fa) R.rt = (int64_t)l; break;
            default: break;
        }
    }
    if (!first) {   // QueryData::init() copied the file's defaults in; the first record starts from None (default_with_params)
        if (R.tol < 0) R.tol = (int64_t)h.tol - 1;
        if (R.tolu < 0) R.tolu = (int64_t)h.tolu - 1;
        if (R.charge < 0) R.charge = (int64_t)h.charge - 1;
    }
    return R;
}

template <int PASS>
__global__ void k_mgf_records(const uint8_t* t, const MgfLine* L, const uint64_t* end_lines, uint64_t n_rec, const MgfHeader* hp, MgfOut o) {
    const MgfHeader h = *hp;
    for (uint64_t r = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; r < n_rec; r += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t l0 = r == 0 ? h.begin_line + 1 : end_lines[r - 1] + 1, l1 = end_lines[r];
        const MgfRecord R = mgf_record(L, l0, l1, r == 0, h);
        const uint64_t per_pep = R.charge >= 0 ? L[R.charge].count : 1;
        const uint64_t id_len = R.title >= 0 ? L[R.title].end - L[R.title].beg : 0;
        const bool kept = id_len > 0 && R.n_pep * per_pep > 0 && R.n_mz > 0 && R.n_mz == R.n_int;
        if (PASS == 0) {
            o.kept[r] = kept;
            o.n_peaks[r] = kept ? R.n_mz : 0;
            o.n_prec[r] = kept ? R.n_pep * per_pep : 0;
            o.id_len[r] = kept ? id_len : 0;
            if (r == n_rec - 1) o.kept[n_rec] = o.n_peaks[n_rec] = o.n_prec[n_rec] = o.id_len[n_rec] = 0;
            continue;
        }
        if (!kept) continue;
        const uint64_t k = o.kept[r], pk = o.n_peaks[r], pr = o.n_prec[r], ib = o.id_len[r];
        o.peak_off[k] = pk;
        o.prec_off[k] = pr;
        o.id_off[k] = ib;
        o.tic[k] = R.tic;
        float rt = 0.0f;
        if (R.rt >= 0) {
            const float s = L[R.rt].a;
            rt = isnan(s) ? raw_quiet(s) : __fdiv_rn(s, 60.0f);
        }
        o.rt[k] = rt;
        uint8_t iso = 0;
        float lo = 0.0f, hi = 0.0f;
        if (R.tol >= 0 && R.tolu >= 0 && L[R.tolu].fa != MGF_UNIT_OTHER) {
            iso = L[R.tolu].fa;
            hi = __uint_as_float(__float_as_uint(L[R.tol].a) & 0x7FFFFFFFu);
            lo = __uint_as_float(__float_as_uint(hi) ^ 0x80000000u);
        }
        const uint64_t tb = R.title >= 0 ? L[R.title].beg : 0;
        for (uint64_t i = 0; i < id_len; i++) o.id_bytes[ib + i] = t[tb + i];
        uint64_t p = pk, q = pr;
        for (uint64_t l = l0; l < l1; l++) {
            const MgfLine& x = L[l];
            if (x.kind == MGF_PEAK && x.fa) {
                o.mz[p] = x.a;
                o.intensity[p] = x.fb ? x.b : 1.0f;
                p++;
            } else if (x.kind == MGF_PEPMASS && x.fa != 2) {
                const float mz = x.fa ? x.a : 0.0f;
                auto put = [&](uint8_t c, uint8_t some) {
                    o.p_mz[q] = mz;
                    o.p_int[q] = x.fb ? x.b : 0.0f;
                    o.p_int_some[q] = x.fb;
                    o.p_charge[q] = c;
                    o.p_charge_some[q] = some;
                    o.p_iso[q] = iso;
                    o.p_lo[q] = lo;
                    o.p_hi[q] = hi;
                    q++;
                };
                if (R.charge >= 0) {
                    const MgfLine& c = L[R.charge];
                    for (uint64_t i = c.beg; i < c.end; i++)
                        if (t[i] >= '0' && t[i] <= '9') put((uint8_t)(t[i] - '0'), 1);
                } else {
                    put(0, 0);
                }
            }
        }
    }
}

// _process: the u32 peak offsets and first-precursor charges k_process_ms2 takes, the largest spectrum, and the first spectrum whose first
// precursor has charge Some(0) (which a u8 charge with 0 = None cannot carry).
__global__ void k_mgf_process_inputs(uint64_t n, const uint64_t* peak_off, const uint64_t* prec_off, const uint8_t* charge, const uint8_t* some,
                                     uint32_t* off32, uint8_t* chg, unsigned int* pmax, unsigned long long* zero_charge) {
    for (uint64_t s = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; s <= n; s += (uint64_t)gridDim.x * blockDim.x) {
        off32[s] = (uint32_t)peak_off[s];
        if (s == n) continue;
        const uint64_t p = prec_off[s];
        chg[s] = some[p] ? charge[p] : 0;
        if (some[p] && charge[p] == 0) atomicMin(zero_charge, (unsigned long long)s);
        atomicMax(pmax, (unsigned int)(peak_off[s + 1] - peak_off[s]));
    }
}

__global__ void k_mgf_counts64(uint64_t n, const uint32_t* cnt, uint64_t* out) {
    const uint64_t s = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (s <= n) out[s] = s < n ? cnt[s] : 0;
}

// k_process_ms2 wrote spectrum s's kept peaks at its raw offset: move them to the compacted offset.
__global__ void k_mgf_compact(uint64_t n, const uint32_t* in_off, const uint32_t* cnt, const float* m, const float* it, const uint64_t* out_off,
                              float* om, float* oi) {
    for (uint64_t s = blockIdx.x; s < n; s += gridDim.x) {
        const uint32_t a = in_off[s], c = cnt[s];
        const uint64_t o = out_off[s];
        for (uint32_t i = threadIdx.x; i < c; i += blockDim.x) {
            om[o + i] = m[a + i];
            oi[o + i] = it[a + i];
        }
    }
}

__global__ void k_mgf_parse_tokens(const uint8_t* bytes, const uint64_t* off, uint64_t n, float* out, uint8_t* ok) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        float v = 0.0f;
        const bool good = mgf_parse_f32(bytes + off[i], off[i + 1] - off[i], &v);
        out[i] = v;
        ok[i] = good;
    }
}

}  // namespace sb
