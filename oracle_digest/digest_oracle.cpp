// digest_oracle.cpp — bulk accessors of the CPU oracle's digest (TEST INFRASTRUCTURE, NOT PRODUCT CODE).
//
// The oracle (oracle/sage_oracle.cpp) restates Parameters::digest; its exports hand out one protein name per ctypes call, too slow to compare
// millions of rows. This file compiles that same restatement (it is included, not copied) and adds:
//   - sod_digest: the digest alone (fasta.rs parse + database.rs:162-258), without the index build;
//   - sizes and export of a peptide table with semi_enzymatic and the protein lists as one CSR of name strings, for a sod_digest handle
//     (sod_*) and for a database built by the oracle's so_db_from_fasta (sod_db_*; same source, same compiler flags, same layout);
//   - sod_auto_chunk_size and sod_prefilter: the database prefilter of runner.rs:104-128, 161-278, composed of the restatement's fasta_parse,
//     digest, build_from_peptides, Scorer::quick_score (with report_psms + 1) and reorder_peptides, with the same table export (sod_pf_*).
#include "../oracle/sage_oracle.cpp"

using namespace so;

static void table_sizes(const std::vector<Peptide>& v, uint64_t* out) {
    uint64_t res = 0, refs = 0, bytes = 0;
    for (const Peptide& p : v) {
        res += p.sequence.size();
        refs += p.proteins.size();
        for (const std::string& s : p.proteins) bytes += s.size();
    }
    out[0] = v.size(); out[1] = res; out[2] = refs; out[3] = bytes;
}

static void table_export(const std::vector<Peptide>& v, uint32_t* seq_off, uint8_t* seq, float* mods, float* nterm, float* cterm, float* mono,
                         uint8_t* decoy, uint8_t* missed, uint8_t* semi, uint64_t* prot_off, uint64_t* name_off, char* names) {
    uint64_t off = 0, ref = 0, nb = 0;
    for (size_t i = 0; i < v.size(); i++) {
        const Peptide& p = v[i];
        seq_off[i] = (uint32_t)off;
        std::memcpy(seq + off, p.sequence.data(), p.sequence.size());
        std::memcpy(mods + off, p.modifications.data(), 4 * p.modifications.size());
        off += p.sequence.size();
        nterm[i] = p.nterm ? *p.nterm : NAN; cterm[i] = p.cterm ? *p.cterm : NAN;
        mono[i] = p.monoisotopic; decoy[i] = p.decoy; missed[i] = p.missed_cleavages; semi[i] = p.semi_enzymatic;
        prot_off[i] = ref;
        for (const std::string& s : p.proteins) {
            name_off[ref++] = nb;
            std::memcpy(names + nb, s.data(), s.size());
            nb += s.size();
        }
    }
    seq_off[v.size()] = (uint32_t)off;
    prot_off[v.size()] = ref;
    name_off[ref] = nb;
}

// Parameters::auto_calculate_prefilter_chunk_size (database.rs:142-160): fasta.digest(&enzyme).len() unmodified peptides, times
// (distinct variable specs + 1) * 2^max_variable_mods, per 2^23 peptides; 0 when targets.len() / chunk_count is 0 (the reference panics).
static uint64_t auto_chunk_size(const BuildParams& P, const Fasta& f) {
    const uint64_t total = fasta_digest(f, P.enzyme).size();
    uint64_t specs = 0;
    for (size_t i = 0; i < P.variable_mods.size(); i++)
        if (i == 0 || P.variable_mods[i - 1].first < P.variable_mods[i].first) specs++;
    const uint64_t chunk_count = (specs + 1) * (1ull << P.max_variable_mods) * total / (1ull << 23);
    return chunk_count == 0 ? f.targets.size() : f.targets.size() / chunk_count;
}

struct Prefiltered {
    std::vector<Peptide> peptides;
    std::vector<uint64_t> rows, kept;   // per chunk
    uint64_t chunk_size = 0, plain = 0;
};

extern "C" {
void* sod_digest(const char* fasta_text, const so_build_params* p) {
    BuildParams P = to_build_params(p);
    Fasta f = fasta_parse(fasta_text, P.decoy_tag, P.generate_decoys);
    return new std::vector<Peptide>(digest(P, f));
}
void sod_free(void* h) { delete (std::vector<Peptide>*)h; }
void sod_sizes(void* h, uint64_t* out) { table_sizes(*(std::vector<Peptide>*)h, out); }
void sod_export(void* h, uint32_t* seq_off, uint8_t* seq, float* mods, float* nterm, float* cterm, float* mono, uint8_t* decoy, uint8_t* missed,
                uint8_t* semi, uint64_t* prot_off, uint64_t* name_off, char* names) {
    table_export(*(std::vector<Peptide>*)h, seq_off, seq, mods, nterm, cterm, mono, decoy, missed, semi, prot_off, name_off, names);
}
void sod_db_sizes(void* db, uint64_t* out) { table_sizes(((DB*)db)->peptides, out); }
void sod_db_export(void* db, uint32_t* seq_off, uint8_t* seq, float* mods, float* nterm, float* cterm, float* mono, uint8_t* decoy, uint8_t* missed,
                   uint8_t* semi, uint64_t* prot_off, uint64_t* name_off, char* names) {
    table_export(((DB*)db)->peptides, seq_off, seq, mods, nterm, cterm, mono, decoy, missed, semi, prot_off, name_off, names);
}

uint64_t sod_auto_chunk_size(const char* fasta_text, const so_build_params* p) {
    BuildParams P = to_build_params(p);
    return auto_chunk_size(P, fasta_parse(fasta_text, P.decoy_tag, P.generate_decoys));
}

// The prefilter of runner.rs:104-128 and 161-278 with chunk_size (0 = automatic) over spectra in so_score_batch's layout (level NULL = all 2).
// Returns NULL when the chunk size is 0 and there are proteins to cut (an empty FASTA is the plain build).
void* sod_prefilter(const char* fasta_text, const so_build_params* p, const so_scorer_params* sp, uint64_t chunk_size, int low_memory, uint64_t min_peaks,
                    uint64_t n, const uint64_t* peak_off, const float* masses, const float* intens, const float* prec_mz, const uint8_t* prec_charge,
                    const float* iso_lo, const float* iso_hi, const float* tic, const uint8_t* level) {
    BuildParams P = to_build_params(p);
    Fasta f = fasta_parse(fasta_text, P.decoy_tag, P.generate_decoys);
    const uint64_t cs = chunk_size ? chunk_size : auto_chunk_size(P, f);
    if (cs == 0 && !f.targets.empty()) return nullptr;
    Prefiltered* h = new Prefiltered();
    h->chunk_size = cs;
    if (cs >= f.targets.size()) {   // runner.rs:110
        h->plain = 1;
        h->peptides = digest(P, f);
        return h;
    }
    so_scorer_params q = *sp;
    q.report_psms += 1;   // runner.rs:191
    std::vector<Spectrum> spectra;
    for (uint64_t i = 0; i < n; i++) {   // runner.rs:252-256
        Spectrum s;
        s.level = level ? level[i] : 2;
        s.n_peaks = (size_t)(peak_off[i + 1] - peak_off[i]);
        if (s.n_peaks < min_peaks || s.level != 2) continue;
        s.has_precursor = !std::isnan(prec_mz[i]);
        s.precursor.mz = prec_mz[i];
        if (prec_charge[i]) s.precursor.charge = prec_charge[i];
        if (iso_lo && iso_hi && !std::isnan(iso_lo[i]) && !std::isnan(iso_hi[i])) s.precursor.isolation_window = Tolerance{DA, iso_lo[i], iso_hi[i]};
        s.masses = masses + peak_off[i];
        s.intensities = intens + peak_off[i];
        s.total_ion_current = tic[i];
        spectra.push_back(s);
    }
    std::vector<Peptide> all;
    for (size_t a = 0; a < f.targets.size(); a += cs) {   // fasta.rs:81-89
        Fasta c;
        c.decoy_tag = f.decoy_tag;
        c.generate_decoys = f.generate_decoys;
        c.targets.assign(f.targets.begin() + a, f.targets.begin() + std::min<size_t>(a + cs, f.targets.size()));
        DB db;
        build_from_peptides(db, digest(P, c), P);
        Scorer sc = make_scorer(&db, &q);
        std::vector<uint8_t> keep(db.peptides.size(), 0);
#pragma omp parallel for schedule(dynamic, 16)   // every mark is a store of 1, as the reference's AtomicBool stores of true
        for (int64_t i = 0; i < (int64_t)spectra.size(); i++) sc.quick_score(spectra[(size_t)i], low_memory != 0, keep.data());
        h->rows.push_back(db.peptides.size());
        uint64_t k = 0;
        for (size_t i = 0; i < db.peptides.size(); i++)
            if (keep[i]) {
                all.push_back(std::move(db.peptides[i]));
                k++;
            }
        h->kept.push_back(k);
    }
    reorder_peptides(all);   // runner.rs:236-238
    h->peptides = std::move(all);
    return h;
}
void sod_pf_free(void* h) { delete (Prefiltered*)h; }
// out: chunk size used, chunk count, plain build; rows / kept: [chunk count] each (may be NULL)
void sod_pf_info(void* h, uint64_t* out, uint64_t* rows, uint64_t* kept) {
    const Prefiltered* x = (const Prefiltered*)h;
    out[0] = x->chunk_size; out[1] = x->rows.size(); out[2] = x->plain;
    for (size_t i = 0; rows && i < x->rows.size(); i++) rows[i] = x->rows[i];
    for (size_t i = 0; kept && i < x->kept.size(); i++) kept[i] = x->kept[i];
}
void sod_pf_sizes(void* h, uint64_t* out) { table_sizes(((Prefiltered*)h)->peptides, out); }
void sod_pf_export(void* h, uint32_t* seq_off, uint8_t* seq, float* mods, float* nterm, float* cterm, float* mono, uint8_t* decoy, uint8_t* missed,
                   uint8_t* semi, uint64_t* prot_off, uint64_t* name_off, char* names) {
    table_export(((Prefiltered*)h)->peptides, seq_off, seq, mods, nterm, cterm, mono, decoy, missed, semi, prot_off, name_off, names);
}
}  // extern "C"
