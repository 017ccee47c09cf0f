// digest_oracle.cpp — bulk accessors of the CPU oracle's digest (TEST INFRASTRUCTURE, NOT PRODUCT CODE).
//
// The oracle (oracle/sage_oracle.cpp) restates Parameters::digest; its exports hand out one protein name per ctypes call, too slow to compare
// millions of rows. This file compiles that same restatement (it is included, not copied) and adds:
//   - sod_digest: the digest alone (fasta.rs parse + database.rs:162-258), without the index build;
//   - sizes and export of a peptide table with semi_enzymatic and the protein lists as one CSR of name strings, for a sod_digest handle
//     (sod_*) and for a database built by the oracle's so_db_from_fasta (sod_db_*; same source, same compiler flags, same layout).
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
}  // extern "C"
