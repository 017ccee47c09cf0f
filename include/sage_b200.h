/* sage_b200.h — C ABI of the H100-native fragment-index search-and-score library.
 *
 * Drop-in boundary for ONE path of lazear/sage (reference @0639176): sage-core's
 *   IndexedDatabase::query / IndexedQuery::page_search   crates/sage/src/database.rs:402-536
 *   Scorer::score (score_standard / score_chimera_fast)   crates/sage/src/scoring.rs:300-767
 * A Rust shim (INTEGRATION.md) keeps `Scorer` / `IndexedDatabase` / `ProcessedSpectrum` as they are and forwards
 * `Scorer::score` / a new `Scorer::score_batch` to these entry points. Plain pointers and sizes only; no C++ or
 * torch types cross this boundary. All functions return 0 on success and a negative SAGE_B200_E* code on failure
 * (never unwind; the reference panics instead — see sage_b200_last_error for the message).
 *
 * Ownership: the caller owns every input/output buffer for the duration of a call; the library copies what it needs
 * to the device and keeps no host pointers. Thread-safety: one sage_b200_scorer may be used by one host thread at a
 * time (calls are serialised internally by a per-scorer mutex); distinct scorers on the same db are independent.
 */
#ifndef SAGE_B200_H
#define SAGE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SAGE_B200_OK 0
#define SAGE_B200_EINVAL (-1)     /* bad argument */
#define SAGE_B200_ECUDA (-2)      /* CUDA runtime error (message has the cudaError string) */
#define SAGE_B200_ENOTMS2 (-3)    /* reference: assert_eq!(query.level, 2)            scoring.rs:301-304 */
#define SAGE_B200_ENOPRECURSOR (-4) /* reference: panic!("missing MS1 precursor")      scoring.rs:466-468 */
#define SAGE_B200_ELIMIT (-5)     /* a documented capacity limit was exceeded */

typedef struct sage_b200_db sage_b200_db;         /* replaces &IndexedDatabase (device-resident)  database.rs:384-395 */
typedef struct sage_b200_scorer sage_b200_scorer; /* replaces Scorer<'db>                          scoring.rs:210-232 */

/* mass.rs:10-16  Tolerance::{Ppm,Pct,Da}(lo,hi) */
enum { SAGE_B200_TOL_PPM = 0, SAGE_B200_TOL_PCT = 1, SAGE_B200_TOL_DA = 2 };
typedef struct { int32_t kind; float lo, hi; } sage_b200_tolerance;

/* ion_series.rs:8-15  Kind */
enum { SAGE_B200_KIND_A = 0, SAGE_B200_KIND_B = 1, SAGE_B200_KIND_C = 2, SAGE_B200_KIND_X = 3, SAGE_B200_KIND_Y = 4, SAGE_B200_KIND_Z = 5 };

/* Peptides as the hot path reads them (peptide.rs:13-31), flattened CSR/SoA. `PeptideIx` == row index. */
typedef struct {
    uint64_t n_peptides;
    const uint32_t* residue_offsets; /* n_peptides+1; residues of peptide i are [off[i], off[i+1]) */
    const uint8_t* sequence;         /* Peptide::sequence bytes, concatenated */
    const float* modifications;      /* Peptide::modifications, parallel to sequence */
    const float* nterm;              /* Peptide::nterm, NaN = None */
    const float* monoisotopic;       /* Peptide::monoisotopic, ascending (database.rs:226-230) */
    const uint8_t* decoy;            /* Peptide::decoy */
    const uint8_t* missed_cleavages; /* Peptide::missed_cleavages */
} sage_b200_peptides;

/* The fragment index exactly as IndexedDatabase holds it (database.rs:378-395). */
typedef struct {
    uint64_t n_fragments;
    const uint32_t* fragment_peptide; /* Theoretical::peptide_index */
    const float* fragment_mz;         /* Theoretical::fragment_mz   */
    uint64_t n_buckets;
    const float* bucket_min;          /* IndexedDatabase::min_value */
    uint64_t bucket_size;             /* IndexedDatabase::bucket_size */
    const uint8_t* ion_kinds;         /* IndexedDatabase::ion_kinds (SAGE_B200_KIND_*) */
    uint64_t n_ion_kinds;
} sage_b200_index;

typedef struct {
    uint64_t n_peptides, n_fragments, n_buckets, bucket_size, n_ion_kinds, total_residues;
    uint64_t device_bytes; /* HBM held by this db */
    int32_t device;
} sage_b200_db_info;

/* Mirror of Scorer's public fields (scoring.rs:210-232). */
typedef struct {
    sage_b200_tolerance precursor_tol, fragment_tol;
    uint16_t min_matched_peaks;
    int8_t min_isotope_err, max_isotope_err;
    uint8_t min_precursor_charge, max_precursor_charge, override_precursor_charge;
    int8_t max_fragment_charge; /* Option<u8>: <0 = None */
    uint8_t chimera, wide_window, annotate_matches;
    uint8_t score_type; /* 0 = SageHyperScore, 1 = OpenMSHyperScore (scoring.rs:10-14) */
    uint32_t report_psms;
} sage_b200_scorer_params;

/* &[ProcessedSpectrum] flattened (spectrum.rs:47-79); only precursors.first() is read (scoring.rs:466). */
typedef struct {
    uint64_t n;
    const uint64_t* peak_offsets;     /* n+1 */
    const float* masses;              /* ProcessedSpectrum::masses (ascending) */
    const float* intensities;         /* ProcessedSpectrum::intensities */
    const float* precursor_mz;        /* Precursor::mz; NaN = spectrum has no precursor */
    const uint8_t* precursor_charge;  /* Precursor::charge; 0 = None */
    const float* isolation_lo;        /* Precursor::isolation_window = Some(Da(lo,hi)); NaN = None. May be NULL (all None) */
    const float* isolation_hi;
    const float* total_ion_current;   /* ProcessedSpectrum::total_ion_current */
    const uint8_t* level;             /* ProcessedSpectrum::level; NULL = all 2 */
    const float* scan_start_time;     /* -> Feature::rt / aligned_rt; NULL = 0 */
    const float* inverse_ion_mobility;/* Precursor::inverse_ion_mobility, NaN/NULL = None -> Feature::ims = 0 */
} sage_b200_spectra;

/* Numeric fields of Feature that the path computes (scoring.rs:69-149, 535-593). spec_id/file_id are re-attached by
 * the caller from `spectrum`; psm_id (global atomic, scoring.rs:163-167) is assigned by the caller after the call. */
typedef struct {
    uint32_t spectrum;      /* index into the batch */
    uint32_t peptide_idx;   /* PeptideIx */
    uint32_t peptide_len;
    uint32_t rank;
    int32_t label;          /* -1 decoy, 1 target */
    float expmass, calcmass;
    uint32_t charge;
    float rt, ims;
    float delta_mass, isotope_error, average_ppm;
    double hyperscore, delta_next, delta_best;
    uint32_t matched_peaks, longest_b, longest_y;
    float longest_y_pct;
    uint32_t missed_cleavages;
    float matched_intensity_pct;
    uint32_t scored_candidates;
    float ms2_intensity;
    double poisson;
    uint32_t fragment_offset, fragment_count; /* into the fragments array when annotate_matches */
} sage_b200_feature;

/* One matched fragment (scoring.rs:152-161, 738-751). */
typedef struct { int32_t kind, charge, ordinal; float intensity, mz_calculated, mz_experimental; } sage_b200_fragment;

/* Work counters of the last score_batch (SURVEY.md §8d algorithmic-bytes terms) + device timings (CUDA events, ms). */
typedef struct {
    uint64_t spectra, peaks, queries, tasks /* (peak,fragment-charge) probes */, pages, entries_scanned, matched_fragments,
        candidates_scored, peptide_record_floats, psms, wide_queries,
        pep_queries /* narrow queries counted peptide-centrically (pages/entries_scanned are then not visited, see DESIGN.md) */, pep_fallbacks,
        wide_overflows /* open-search queries whose survivor list overflowed (replayed inside the counting kernel) */;
    uint64_t algorithmic_bytes;    /* SURVEY.md §8d formula, whole batch */
    uint64_t prelim_bytes;         /* the part of it the preliminary-scoring kernel(s) move: peak masses, bucket / page probes, entries scanned */
    uint64_t score_bytes;          /* the part k_score moves: peak intensities, candidate peptide records, PSM rows */
    uint64_t h2d_bytes, d2h_bytes; /* bytes copied across PCIe for the batch */
    uint64_t kernel_launches;
    uint64_t chunk_retries;        /* chunks re-run because a device work list was sized too small (first batches of a scorer; see DESIGN.md) */
    float ms_total, ms_h2d, ms_setup, ms_prelim, ms_score, ms_d2h; /* summed over chunks */
    float ms_prelim_count;         /* the part of ms_prelim before the heap-replay kernels: k_prelim_narrow_warp + k_prelim_narrow */
    float ms_wall;                 /* host wall clock of the last score_batch call, entry to return (includes every copy and wait) */
} sage_b200_counters;

int sage_b200_device_count(void);

/* IndexedDatabase -> device. `index` as built by Parameters::build (database.rs:260-365). */
int sage_b200_db_create(const sage_b200_peptides* peptides, const sage_b200_index* index, int device, sage_b200_db** out);

/* Parameters::build_from_peptides on the device (database.rs:265-365): fragment generation for `ion_kinds` with the
 * `min_ion_index` filter, global sort by fragment m/z, bucketing, per-bucket sort by PeptideIx. */
int sage_b200_db_build(const sage_b200_peptides* peptides, uint64_t bucket_size, const uint8_t* ion_kinds, uint64_t n_ion_kinds,
                       uint64_t min_ion_index, int device, sage_b200_db** out);

int sage_b200_db_get_info(const sage_b200_db* db, sage_b200_db_info* info);
/* Copies the index back in the reference layout (IndexedDatabase::fragments / min_value); any pointer may be NULL. */
int sage_b200_db_export_index(const sage_b200_db* db, uint32_t* fragment_peptide, float* fragment_mz, float* bucket_min);
void sage_b200_db_destroy(sage_b200_db* db);

int sage_b200_scorer_create(const sage_b200_db* db, const sage_b200_scorer_params* params, sage_b200_scorer** out);
void sage_b200_scorer_destroy(sage_b200_scorer* scorer);
/* Tuning knobs that do not change results.
 *   "pep_cap"         precursor windows with at most this many peptides are counted by streaming the candidates' ion tables instead of
 *                     probing the fragment index (default 0 = always probe the index, the reference's loop order)
 *   "sort_spectra"    1 (default): process spectra in ascending precursor order for cache locality; results are returned in input order
 *   "pipeline_chunks" cut every batch into at least this many pipelined chunks (default 1: chunks of <= 65536 spectra)
 *   "narrow_index"    1 (default): narrow precursor windows (up to 8192 peptides) are counted against a second, peptide-block-major copy of the
 *                     fragment index (one short m/z run per probe); 0: the reference's loop order against the page index — identical results,
 *                     and the only mode that fills the counters `pages` / `entries_scanned` (the reference algorithm's work terms)
 *   "score_split"     1 (default): non-chimeric scoring runs as three kernels (match per spectrum; fold and rank / rows one thread per candidate);
 *                     0: one fused kernel per spectrum (always used for chimera, annotate_matches, quick_score) — identical results
 *   "mass_parts"      1..4 (default 2): the peak-mass copy of a chunk from PINNED caller memory is cut into this many runs of spectra and the
 *                     counting kernel is queued once per run, so it starts while the rest of the copy is in flight
 *   "wide_tile", "wide_lmax", "worklist_reset", "narrow_block"   test hooks (tile size / survivor-list size of the open-search kernel; forget learned
 *                     list sizes; peptides per block of the narrow-search copy, 0 = sized by the average precursor window, else 64..65536) */
int sage_b200_scorer_set_option(sage_b200_scorer* scorer, const char* name, int64_t value);

/* Scorer::score over a batch (runner.rs:311-325 `par_iter().flat_map(|s| scorer.score(s))`).
 * features: caller-allocated, n * report_psms entries; spectrum i's PSMs are features[i*report_psms .. +counts[i]).
 * fragments/fragment_capacity/fragments_used: only with annotate_matches (may be NULL otherwise). */
int sage_b200_score_batch(sage_b200_scorer* scorer, const sage_b200_spectra* spectra, sage_b200_feature* features, uint32_t* counts,
                          sage_b200_fragment* fragments, uint64_t fragment_capacity, uint64_t* fragments_used);

/* Same result as sage_b200_score_batch, computed by several GPUs of one box from one host process: contiguous blocks of spectra go to
 * scorers[0..n) (one per device, each on its own index replica, one host thread each); no collective. annotate_matches is not supported here. */
int sage_b200_score_batch_multi(sage_b200_scorer* const* scorers, int n_scorers, const sage_b200_spectra* spectra, sage_b200_feature* features,
                                uint32_t* counts);

/* Pins the calling host thread to the CPUs of the NUMA node next to `device` (PCI topology from sysfs): call it on the thread that will
 * allocate pinned buffers for and submit batches to that GPU (score_batch_multi does it for its own worker threads; a rayon pool would do it in
 * its start handler). Returns the NUMA node, or -1 when the topology is unknown (nothing changed). */
int sage_b200_bind_thread_to_device(int device);

/* Scorer::quick_score over a batch (scoring.rs:255-298; prefilter of runner.rs:143-278). keep has one byte per peptide of the db and is
 * OR-ed (the reference stores `true` into &[AtomicBool]). prefilter_low_memory selects the branch of scoring.rs:270. */
int sage_b200_quick_score(sage_b200_scorer* scorer, const sage_b200_spectra* spectra, int prefilter_low_memory, uint8_t* keep);

/* The same call split in phases for device-resident reuse (one batch of <= 262144 spectra / 2^26 peaks):
 * upload makes the spectra resident in HBM, run launches the kernels (results stay on the device; may be repeated),
 * download copies the Feature rows back. score_batch == upload + run + download per chunk. */
int sage_b200_batch_upload(sage_b200_scorer* scorer, const sage_b200_spectra* spectra);
int sage_b200_batch_run(sage_b200_scorer* scorer);
int sage_b200_batch_download(sage_b200_scorer* scorer, sage_b200_feature* features, uint32_t* counts);

/* Scorer::initial_hits for one spectrum (scoring.rs:418-462): the preliminary list in the reference's heap order.
 * White-box hook used by the parity tests. Returns the list length (<= cap written) or a negative error. */
int64_t sage_b200_initial_hits(sage_b200_scorer* scorer, const sage_b200_spectra* one_spectrum, uint16_t* matched, uint32_t* peptide,
                               uint8_t* charge, int8_t* isotope_error, uint64_t cap, uint64_t* matched_peaks, uint64_t* scored_candidates);

int sage_b200_counters_get(const sage_b200_scorer* scorer, sage_b200_counters* out);

/* SpectrumProcessor (spectrum.rs:39-44, 263-412) for centroided MS2 spectra — the step right before the hot path (SURVEY.md §8 row f2). */
typedef struct { uint64_t take_top_n; uint8_t deisotope; float min_deisotope_mz; } sage_b200_processor_params;
typedef struct {                    /* &[RawSpectrum] flattened (spectrum.rs:81-106) */
    uint64_t n;
    const uint64_t* peak_offsets;   /* n+1 */
    const float* mz;                /* RawSpectrum::mz (ascending) */
    const float* intensity;         /* RawSpectrum::intensity */
    const uint8_t* precursor_charge;/* precursors.first().charge, 0 = None (deisotoping then assumes up to 3+, spectrum.rs:289-293) */
    const uint8_t* level;           /* ms_level; NULL = all 2; other levels are rejected */
} sage_b200_raw_spectra;
/* process(): out_peak_offsets[n+1]; out_masses / out_intensities sized for the raw peak count (at most min(raw, take_top_n) are kept per spectrum);
 * out_tic[n] = ProcessedSpectrum::total_ion_current. */
int sage_b200_process_spectra(int device, const sage_b200_processor_params* processor, const sage_b200_raw_spectra* raw, uint64_t* out_peak_offsets,
                              float* out_masses, float* out_intensities, float* out_tic);

/* A batch of RawSpectrum of any MS level (spectrum.rs:81-106) flattened. */
typedef struct {
    uint64_t n;
    const uint64_t* peak_offsets;   /* n+1 */
    const float* mz;                /* RawSpectrum::mz, in any order */
    const float* intensity;
    const uint8_t* level;           /* ms_level, required */
    const uint8_t* precursor_charge;/* read for level 2 only (as in sage_b200_raw_spectra); may be NULL when no spectrum is level 2 */
    const float* mobility;          /* per raw peak; NULL = no spectrum of the batch has mobility (the convention of sage_b200_ms1) */
} sage_b200_raw_batch;
/* SpectrumProcessor::process (spectrum.rs:338-412) for every level: level 2 as sage_b200_process_spectra (same kernel, same ELIMIT past its
 * shared-memory budget); other levels keep every peak, mass = mz - PROTON, stably sorted by total_cmp, with no size limit per spectrum.
 * Outputs are sized for the raw peak count and compacted: out_peak_offsets[n+1]; out_mobilities parallel to out_masses, holding the sorted
 * mobilities of level-1 spectra when raw->mobility is set, NaN for every other spectrum (whose ProcessedSpectrum::mobilities is empty);
 * out_tic[n]. Bit for bit the reference's result on x86-64, NaNs included (DESIGN.md §16). */
int sage_b200_process_raw(int device, const sage_b200_processor_params* processor, const sage_b200_raw_batch* raw, uint64_t* out_peak_offsets,
                          float* out_masses, float* out_intensities, float* out_mobilities, float* out_tic);

/* tmt::find_reporter_ions (tmt.rs:193-211) over a batch: out[i * n_labels + l] = intensity of the most intense peak of spectrum i within
 * label_tolerance of labels[l] (offset -PROTON, as the reference), 0 where none (the unwrap_or_default of tmt::quantify, tmt.rs:333). */
int sage_b200_find_reporter_ions(int device, uint64_t n, const uint64_t* peak_offsets, const float* masses, const float* intensities, const float* labels,
                                 uint64_t n_labels, sage_b200_tolerance label_tolerance, float* out);

/* Which build of glibc's log() the host libm is (replaces Rust's f64::ln, scoring.rs:179-201 / :512): the kernels reproduce that function
 * operation by operation so that hyperscore, poisson and ranks under near-ties carry the same bits as the CPU path on this host.
 * 0 = x86-64 glibc on a CPU with FMA+AVX2 (`__log_fma`), 1 = the uncontracted build (`__log_sse2`/`__log_avx`, musl, aarch64),
 * -1 = neither matched std::log on the probe inputs (the device then uses variant 0; f64 fields agree to <= 1 ulp). */
int sage_b200_host_log_variant(void);
/* 1 when the host libm's log1pf (Rust's f32::ln_1p: OpenMS hyperscore, scoring.rs:190-197) is the glibc / fdlibm function the kernels reproduce. */
int sage_b200_host_log1pf_exact(void);
/* Test hook: out[i] = the device's evaluation of log(x[i]) with `variant` (0/1), or of (double)log1pf((float)x[i]) with variant 2 — compared bit for bit with the host libm by tests/test_glibc_log.py. */
int sage_b200_device_log(int device, int variant, const double* x, uint64_t n, double* out);

/* ---------------------------------------------------------------------------------------------------------------------------------------------
 * Label-free quantification (lfq.rs): build_feature_map (lfq.rs:94-193) and FeatureMap::quantify (lfq.rs:226-304) on the device.
 * create -> add_ms1 (any number of batches; the result does not depend on how spectra are split) -> integrate. Calls on one handle are
 * serialised by a per-handle mutex. Grid cells are summed in a defined order (batches in call order, spectra in input order, peaks in order,
 * lo before hi contribution), so every cell is reproducible bit for bit; see DESIGN.md §9 for the exactness contract.
 */
typedef struct sage_b200_lfq sage_b200_lfq;   /* replaces FeatureMap + the DashMap<(PrecursorId, bool), Grid> of quantify */

/* lfq.rs:25-37 */
enum { SAGE_B200_PEAK_RETENTION_TIME = 0, SAGE_B200_PEAK_SPECTRAL_ANGLE = 1, SAGE_B200_PEAK_INTENSITY = 2, SAGE_B200_PEAK_HYBRID = 3 };
enum { SAGE_B200_INTEGRATE_APEX = 0, SAGE_B200_INTEGRATE_SUM = 1 };

/* LfqSettings (lfq.rs:45-54) plus Search::precursor_charge (min, max). */
typedef struct {
    int32_t peak_scoring;         /* SAGE_B200_PEAK_* */
    int32_t integration;          /* SAGE_B200_INTEGRATE_* */
    double spectral_angle;
    float ppm_tolerance, mobility_pct_tolerance, peptide_q_value;
    uint8_t combine_charge_states;
    uint8_t min_precursor_charge, max_precursor_charge;
} sage_b200_lfq_params;

/* The Feature fields build_feature_map reads, n rows in the caller's confidence order (rows with peptide_q <= peptide_q_value && label == 1
 * are kept; the first kept row of each peptide wins, lfq.rs:100-131). */
typedef struct {
    uint64_t n;
    const uint32_t* peptide_idx;
    const float* peptide_q;
    const int32_t* label;
    const float* aligned_rt;
    const float* calcmass;
    const uint32_t* file_id;      /* < n_files */
    const float* ims;
} sage_b200_lfq_features;

/* retention_alignment.rs:87-93 (file_id is the array position) */
typedef struct { float max_rt, slope, intercept; } sage_b200_alignment;

/* One batch of MS1 ProcessedSpectrum (spectrum.rs:58-79). */
typedef struct {
    uint64_t n;
    const uint64_t* peak_offsets;     /* n+1 */
    const float* masses;              /* ProcessedSpectrum::masses (mz - PROTON), ascending */
    const float* intensities;
    const uint32_t* file_id;          /* < n_files */
    const float* scan_start_time;
    const float* mobilities;          /* per peak; NULL = no spectrum of the batch has mobilities */
} sage_b200_ms1;

/* PrecursorRange (lfq.rs:70-82) as the sorted feature map holds it. */
typedef struct {
    float rt, mass_lo, mass_hi, mobility_lo, mobility_hi;
    uint32_t peptide, file_id;
    uint8_t charge, isotope, decoy, _pad;
} sage_b200_lfq_range;

/* One entry of quantify's map: key (PrecursorId, decoy), Peak (lfq.rs:335-345); areas are returned in a separate [rows x n_files] array. */
typedef struct {
    uint32_t peptide;
    uint8_t charge;                   /* PrecursorId::Charged; 0 for PrecursorId::Combined */
    uint8_t decoy;
    uint16_t _pad0;
    uint32_t rt;                      /* Peak::rt, bin 0..99 */
    uint32_t _pad1;
    double spectral_angle, score;
} sage_b200_lfq_row;

typedef struct {
    uint64_t n_peptides;              /* peptides that passed the filter (one PrecursorRange seed each) */
    uint64_t n_ranges, n_pages, n_grids /* upper bound of integrate's row count */, n_files;
    uint64_t grids_touched, ms1_spectra, ms1_peaks, contributions;
    uint64_t device_bytes;
    float ms_build, ms_trace, ms_integrate, ms_download;   /* CUDA events: create, summed add_ms1, last integrate's kernels and copy-back */
} sage_b200_lfq_info;

/* build_feature_map. `peptides` is the table the db was built from (only residue_offsets and sequence are read: carbon / sulfur counts,
 * mass.rs:78-116); alignments has n_files entries. EINVAL for a file_id >= n_files or a peptide_idx outside the db; ELIMIT when the grids
 * (n_grids * n_files * 300 f64) do not fit the device's free memory (checked before allocating). */
int sage_b200_lfq_create(const sage_b200_db* db, const sage_b200_peptides* peptides, const sage_b200_lfq_params* params,
                         const sage_b200_lfq_features* features, uint64_t n_files, const sage_b200_alignment* alignments, sage_b200_lfq** out);
/* The tracing loop of quantify (lfq.rs:239-287) over one batch. EINVAL for a file_id >= n_files. */
int sage_b200_lfq_add_ms1(sage_b200_lfq* lfq, const sage_b200_ms1* ms1);
/* One batch of raw MS1 RawSpectrum: mz in any order. */
typedef struct {
    uint64_t n;
    const uint64_t* peak_offsets;     /* n+1 */
    const float* mz;
    const float* intensity;
    const uint32_t* file_id;          /* < n_files */
    const float* scan_start_time;
    const float* mobility;            /* per raw peak; NULL = no spectrum of the batch has mobility */
} sage_b200_raw_ms1;
/* add_ms1 of the batch SpectrumProcessor::process makes of raw_ms1: the spectra are processed on the device (as sage_b200_process_raw does
 * level 1) and traced there; the processed peaks never cross PCIe. Bit for bit equal to add_ms1 of the processed batch. */
int sage_b200_lfq_add_raw_ms1(sage_b200_lfq* lfq, const sage_b200_raw_ms1* raw_ms1);
/* summarize_traces + integrate (lfq.rs:447-610) for every touched grid: rows ordered by (id, decoy); areas[row * n_files + file].
 * capacity >= info.n_grids always suffices; *n_rows receives the row count. */
int sage_b200_lfq_integrate(sage_b200_lfq* lfq, sage_b200_lfq_row* rows, double* areas, uint64_t capacity, uint64_t* n_rows);
int sage_b200_lfq_get_info(sage_b200_lfq* lfq, sage_b200_lfq_info* info);
/* Test hook: the sorted ranges (n_ranges), min_rts (n_pages), and optionally the raw grid matrices (n_grids * n_files * 3 * 100 f64, grid g
 * at [g * n_files * 300], row file * 3 + isotope) and their touched flags (n_grids). Grid g is (peptide slot, [charge,] decoy) in ascending
 * (PeptideIx, charge, decoy) order. Any pointer may be NULL. */
int sage_b200_lfq_export(sage_b200_lfq* lfq, sage_b200_lfq_range* ranges, float* min_rts, double* grids, uint8_t* touched);
void sage_b200_lfq_destroy(sage_b200_lfq* lfq);

/* ---------------------------------------------------------------------------------------------------------------------------------------------
 * PSM rescoring (runner.rs:280-291 spectrum_fdr): linear_discriminant::score_psms (mass-error KDE, 20-feature LDA, discriminant KDE and
 * posterior errors), the heuristic fallback when it returns None, the descending sort and qvalue::spectrum_q_value. Every output is
 * reproducible bit for bit under the orders of DESIGN.md §10.
 */
typedef struct { sage_b200_tolerance precursor_tol; } sage_b200_fdr_params;   /* Ppm or Da; Pct -> EINVAL (linear_discriminant.rs:142) */
typedef struct {
    float* discriminant_score;       /* [n], indexed like the input rows */
    float* posterior_error;          /* [n] log10(PEP) as f32, -324 for PEP 0; 1.0 when the LDA was not fitted (scoring.rs:577) */
    float* spectrum_q;               /* [n] */
    uint32_t* order;                 /* [n] input row at each sorted position (descending discriminant, ties by ascending input row) */
    uint64_t passing;                /* spectrum_q_value's return: rows with q <= 0.01 (targets and decoys) */
    int32_t lda_fitted;              /* 0: score_psms returned None and the heuristic was used */
    double coef[20];                 /* the LDA weights when Gauss::solve succeeded (also when they are not finite, which falls back); else 0 */
    double eps;                      /* the Gauss::solve ridge that succeeded; 0 when none did or the LDA was not trained */
    float ms_mass_kde, ms_features, ms_lda, ms_discriminant_kde, ms_sort_q, ms_total;   /* CUDA-event stage times of the call */
} sage_b200_fdr_out;
/* rows: the Feature rows the search returned, in the caller's order. aligned_rt / delta_rt_model / delta_ims_model: [n] each, or NULL for the
 * Feature defaults (scoring.rs:583-585: aligned_rt = rt, 0.999 for both deltas). EINVAL for a Pct or unknown tolerance; ELIMIT beyond
 * 65535 * 4096 rows (the KDE's chunk grid), for a tolerance span of 2^24 or more mass-error bins, or when the work buffers do not fit the device's
 * free memory (checked before allocating). */
int sage_b200_spectrum_fdr(int device, const sage_b200_fdr_params* p, const sage_b200_feature* rows, uint64_t n, const float* aligned_rt,
                           const float* delta_rt_model, const float* delta_ims_model, sage_b200_fdr_out* out);
/* White-box hook: kde::Builder::build (kde.rs:83-136) with bins, monotonic and bw_adjust = x * bw_factor; scores f64[n], decoy u8[n] (nonzero =
 * decoy). out_bins[bins] is the PEP per bin; *min_score and *score_step place the bins. ELIMIT beyond 2^31 - 1 scores or 2^24 bins. */
int sage_b200_kde_build(int device, const double* scores, const uint8_t* decoy, uint64_t n, uint64_t bins, int monotonic, double bw_factor,
                        double* out_bins, double* min_score, double* score_step);
/* Test hook: out[i] = the device's evaluation of glibc's exp (function 0), log1p (1) or log10 (2) at x[i]; variant 0 = the FMA builds,
 * 1 = the uncontracted builds, -1 = the variant the library selected for this host's libm. */
int sage_b200_device_math(int device, int function, int variant, const double* x, uint64_t n, double* out);

/* ---------------------------------------------------------------------------------------------------------------------------------------------
 * Retention-time alignment and RT / mobility prediction (runner.rs:513-531 predict_rt): the ascending poisson sort and interim
 * qvalue::spectrum_q_value, retention_alignment::global_alignment, retention_model::predict and mobility_model::predict (regression.rs's
 * LinearRegression::fit). Every output is reproducible bit for bit under the orders of DESIGN.md §11. The rows are not reordered.
 */
typedef struct {
    float* aligned_rt;                /* [n] Feature::aligned_rt */
    float* predicted_rt;              /* [n] clamp(0, 1); 0.0 when the RT model was not fitted */
    float* delta_rt_model;            /* [n] |aligned_rt - predicted_rt|; 0.999 when the RT model was not fitted */
    float* predicted_ims;             /* [n] clamp(0, 2); 0.0 when the mobility model was not fitted */
    float* delta_ims_model;           /* [n] |ims - predicted_ims|; 0.999 when the mobility model was not fitted */
    float* spectrum_q;                /* [n] or NULL: the interim q-values, computed over the ascending-poisson order, indexed like the rows */
    sage_b200_alignment* alignments;  /* [n_files] global_alignment's result, file_id = position; the input of sage_b200_lfq_create */
    uint64_t training_rows;           /* rows with label == 1 && q <= 0.01 */
    uint64_t aligned_peptides;        /* matrix rows kept (peptides whose mean normalised RT is_normal) */
    int32_t rt_fitted;                /* 0: LinearRegression::fit returned None (no training rows, or Gauss::solve failed at every eps) */
    double rt_r2, rt_eps, rt_beta[69];/* r2 = 1 - sse / y_var, the Gauss::solve ridge that succeeded, the coefficients; 0 when not fitted */
    int32_t ims_fitted;
    double ims_r2, ims_eps, ims_beta[100];
    float ms_sort_q, ms_alignment, ms_rt_model, ms_ims_model, ms_total;   /* CUDA-event stage times of the call (the host solves included) */
} sage_b200_rt_out;
/* rows: the Feature rows in the caller's order; file_id[n] < n_files; peptides: the table the db was built from (residue_offsets, sequence and
 * monoisotopic are read). EINVAL for a file_id >= n_files, a peptide_idx outside the db, n_files == 0 with rows, a peptide table of another size
 * than the db's, or a residue byte outside 'A'..'Z' in a referenced peptide; ELIMIT beyond 2^31 - 1 rows or when the work buffers (the
 * peptide x file matrix the largest) do not fit the device's free memory (checked before allocating). n == 0: every alignment is
 * {0, 1, 0} and nothing is fitted. */
int sage_b200_predict_rt(const sage_b200_db* db, const sage_b200_peptides* peptides, const sage_b200_feature* rows, const uint32_t* file_id, uint64_t n,
                         uint64_t n_files, sage_b200_rt_out* out);

/* ---------------------------------------------------------------------------------------------------------------------------------------------
 * Picked FDR (fdr.rs): picked_peptide and picked_protein (runner.rs:534-537, Competition::assign_q_value) and picked_precursor (runner.rs:572).
 * Every output is reproducible bit for bit under the definitions of DESIGN.md §12; competition entries are ordered by the first row that
 * reaches them, so call these on the rows in spectrum_fdr's sorted order, as the runner does.
 */
typedef struct {
    const float* cterm;               /* [n_peptides] Peptide::cterm, NaN = None; NULL = None for every peptide */
    const uint32_t* n_proteins;       /* [n_peptides] Peptide::proteins.len() */
    const uint32_t* protein;          /* [n_peptides] id of the single protein name (equal ids <=> equal names); read only where n_proteins == 1 */
    uint8_t generate_decoys;          /* IndexedDatabase::generate_decoys */
} sage_b200_picked_params;
typedef struct {
    float* peptide_q;                 /* [n] indexed like the rows */
    float* protein_q;                 /* [n]; 1.0 for rows whose peptide has != 1 protein */
    uint64_t peptide_passing, protein_passing;   /* assign_q_value's return values: target rows at q <= 0.01 */
    uint64_t peptide_entries, protein_entries;   /* competition entries (the maps' sizes) */
    float ms_keys, ms_peptide, ms_protein, ms_total;   /* CUDA-event stage times: peptide keys, each competition, the whole call */
} sage_b200_picked_out;
/* picked_peptide then picked_protein over the rows. peptides: the table the rows' PeptideIx index (residue_offsets, sequence, modifications,
 * nterm and decoy are read; the decoy flag is Peptide::decoy). The call takes no db handle: the caller passes the same table the searched db
 * was built from (sage_b200_db_create / _build), since a PeptideIx means nothing against another table; only its size is checked here, through
 * the PeptideIx bound. picked_protein's Ix is (protein, side) with generate_decoys and the protein alone without; the reference's Ix is the
 * string `decoy_tag + name`, so a target protein whose name starts with the decoy tag would share an Ix with a decoy there, and not here. EINVAL for a null required pointer, a peptide_idx outside the table, or two
 * distinct peptides on one side with one key (the reference panics; the message names both PeptideIx); ELIMIT beyond 2^31 - 1 rows, beyond
 * 65535 * 4096 rows (the KDE's chunk grid) or when the work buffers do not fit the device's free memory (checked before allocating).
 * n == 0: no device work. */
int sage_b200_picked_fdr(int device, const sage_b200_peptides* peptides, const sage_b200_picked_params* p, const sage_b200_feature* rows,
                         const float* discriminant_score, uint64_t n, sage_b200_picked_out* out);
/* picked_precursor over quantify's rows in sage_b200_lfq_integrate's order: score = Peak::score, decoy (nonzero = decoy). q_value[n] is
 * indexed like the rows; *passing counts target rows at q <= 0.05. EINVAL for a null pointer; ELIMIT beyond 2^31 - 1 rows or when the work
 * buffers do not fit the device's free memory (checked before allocating). n == 0: no device work. */
int sage_b200_picked_precursor(int device, const double* score, const uint8_t* decoy, uint64_t n, float* q_value, uint64_t* passing);
/* White-box hook: entry_rank[i] = the rank, in first-appearance order, of row i's picked_peptide entry. hash_bits (3..64) truncates the key
 * hash so that distinct keys collide and the exact comparison that separates them is exercised; with hash_bits < 64 at most 2^16 rows
 * (ELIMIT beyond: equal-hash runs are compared pairwise). */
int sage_b200_competition_keys(int device, const sage_b200_peptides* peptides, const sage_b200_picked_params* p, const uint32_t* peptide_idx, uint64_t n,
                               uint32_t hash_bits, uint32_t* entry_rank);

/* ---------------------------------------------------------------------------------------------------------------------------------------------
 * Protein grouping and picked protein-group FDR (protein_grouping.rs generate_protein_groups, fdr.rs picked_protein_group; runner.rs:513-572).
 * Every output is reproducible exactly under the definitions of DESIGN.md §13:
 *   - a protein name is an id (equal ids <=> equal names). Names containing '/' or ';', and a target name that starts with the decoy tag,
 *     are not modelled: the first change the reference's strings and group counts, the second makes a target and a tagged decoy share a key;
 *   - pass 1 uses threshold.clamp(0, 1) (NaN stays NaN and selects nothing), pass 2 uses 1.0; a pass annotates only rows still unannotated;
 *   - competition entries are ordered by the first row that reaches them: call this on the rows in spectrum_fdr's sorted order.
 * Strings are not built here. The caller builds the reference's `protein_groups` string of row i from the outputs:
 *   - pass[i] > 0: for each group g in row_groups[row_group_offsets[i] .. row_group_offsets[i+1]), the member names of g, each written
 *     decoy_tag + name when group_decoy[g] && generate_decoys, sorted and joined with '/'; these group strings sorted and joined with ';';
 *   - pass[i] == 0 (fallback): Peptide::proteins(decoy_tag, generate_decoys), the peptide's names in stored order joined with ';', each
 *     written decoy_tag + name when the peptide is a decoy and generate_decoys is set.
 */
typedef struct {
    const uint32_t* protein_offsets;  /* [n_peptides + 1] peptide p's proteins are protein_ids[protein_offsets[p] .. protein_offsets[p+1]) */
    const uint32_t* protein_ids;      /* Peptide::proteins as name ids, in stored order (a repeated name stays repeated); each < n_names */
    uint64_t n_names;
    uint8_t protein_grouping;         /* 0: no grouping, every row takes the fallback */
    uint8_t has_threshold;            /* 1: Some(threshold), two passes; 0: None, pass 2 only */
    uint8_t generate_decoys;          /* IndexedDatabase::generate_decoys */
    float threshold;                  /* the confident peptide q-value threshold of pass 1 */
} sage_b200_protein_group_params;
typedef struct {
    uint32_t* num_protein_groups;     /* [n] Feature::num_protein_groups */
    float* protein_group_q;           /* [n] Feature::protein_group_q: 1.0 for rows with num_protein_groups != 1 */
    uint8_t* pass;                    /* [n] the pass that annotated the row: 1 or 2, 0 = fallback */
    uint64_t* row_group_offsets;      /* [n + 1] */
    uint32_t* row_groups;             /* [row capacity] each annotated row's covered groups, ascending; fallback rows have none.
                                         row capacity = the sum over rows of their peptide's protein count */
    uint64_t* group_offsets;          /* [group capacity + 1] the group tables of pass 1 then pass 2, concatenated; group g of pass 2 is
                                         groups[0] + g. group capacity = 2 * min(protein_offsets[n_peptides], 2 * n_names) */
    uint32_t* group_members;          /* [group capacity] name ids of each group, ascending */
    uint8_t* group_covered;           /* [group capacity] 1: the group is in the cover */
    uint8_t* group_decoy;             /* [group capacity] the decoy flag of the group's (name, decoy) keys */
    uint64_t peptides[2];             /* per pass: distinct PeptideIx in the pass's peptide set */
    uint64_t proteins[2];             /* per pass: distinct (name, decoy) keys (ProteinIx) */
    uint64_t meta_peptides[2], groups[2], edges[2];
    uint64_t covered[2];              /* groups in the cover */
    uint64_t forced[2];               /* groups forced in by a peptide of degree 1 */
    uint64_t greedy_picks[2];         /* add_largest_to_cover picks */
    uint64_t components[2];           /* connected components left after the forced picks */
    uint64_t largest_component[2];    /* groups in the largest of them */
    uint64_t annotated[2];            /* rows annotated by the pass */
    uint64_t passing;                 /* picked_protein_group's return: target rows at q <= 0.01 */
    uint64_t entries;                 /* picked_protein_group's competition entries */
    float ms_build[2], ms_cover[2], ms_lookup[2], ms_picked, ms_total;   /* CUDA-event stage times of the call */
} sage_b200_protein_group_out;
/* generate_protein_groups(db, rows, protein_grouping, has_threshold ? Some(threshold) : None) then picked_protein_group. rows: the Feature
 * rows (peptide_idx and label are read); peptide_q and discriminant_score: [n] each, indexed like the rows; peptides: the table the rows'
 * PeptideIx index (only n_peptides and decoy are read). The group set of a pass reads the label (label != -1); the lookup and the
 * competition side read Peptide::decoy, as the reference does. EINVAL for a null required pointer, a peptide_idx outside the table,
 * protein_offsets not starting at 0 or decreasing, or a protein id >= n_names; ELIMIT beyond 2^31 - 1 rows, 65535 * 4096 rows (the KDE's chunk
 * grid), 2^30 names or 2^31 - 1 protein entries, or when the work buffers do not fit the device's free memory (checked before allocating).
 * The argument checks run before the device is looked at. n == 0: no device work. */
int sage_b200_protein_groups(int device, const sage_b200_peptides* peptides, const sage_b200_protein_group_params* p, const sage_b200_feature* rows,
                             const float* peptide_q, const float* discriminant_score, uint64_t n, sage_b200_protein_group_out* out);
/* Test hook: BipartiteGraph::new(edges, n_left, n_right).into_cover() (protein_grouping.rs) on the device, edge k = (left[k], right[k]);
 * parallel edges allowed. cover[n_left] receives 1 for each left node in the cover. EINVAL for a null pointer or an endpoint out of range;
 * ELIMIT beyond 2^31 - 1 edges or nodes. */
int sage_b200_bipartite_cover(int device, const uint32_t* left, const uint32_t* right, uint64_t n_edges, uint64_t n_left, uint64_t n_right,
                              uint8_t* cover);

/* ---------------------------------------------------------------------------------------------------------------------------------------------
 * Digest (Parameters::digest, database.rs:162-258): FASTA text -> the sorted, merged peptide table with its protein lists, in PeptideIx order.
 * The FASTA is parsed on the host (fasta.rs:14-56, one pass); cleavage, windows, per-protein de-duplication, grouping, modification
 * enumeration, the sort and the merge run on the device. The table is the reference's bit for bit under the definitions of DESIGN.md §14;
 * the parameters are normalised as Builder does: max_variable_mods is raised to 1, invalid mod specs are skipped, static specs are ordered
 * by spec (a repeated spec: the last mass wins), variable (spec, mass) pairs are stable-sorted by spec.
 * create -> get_info (the sizes) -> export (caller-allocated arrays) -> destroy.
 */
typedef struct sage_b200_digest sage_b200_digest;

/* Builder (database.rs:17-41) without the index fields. */
typedef struct {
    uint8_t missed_cleavages;
    uint64_t min_len, max_len;                /* max_len <= 255 (the library's peptide-length limit) */
    const char* cleave_at;                    /* "" = non-specific (missed cleavages taken as 0), "$" = no cleavage; NULL = "" */
    const char* restrict_;                    /* NULL = "" */
    uint8_t c_terminal, semi_enzymatic;
    float peptide_min_mass, peptide_max_mass; /* inclusive */
    const char* const* static_specs;          /* "C", "^", "[", "$", "]", "^Q", ...; n_static entries */
    const float* static_masses;
    uint64_t n_static;
    const char* const* variable_specs;        /* one entry per (spec, mass) */
    const float* variable_masses;
    uint64_t n_variable;
    uint64_t max_variable_mods;               /* <= 8 */
    const char* decoy_tag;                    /* NULL = "rev_" */
    uint8_t generate_decoys;
} sage_b200_digest_params;

typedef struct {
    uint64_t n_peptides, n_residues, n_protein_refs, n_names, name_bytes;   /* the export's array sizes */
    uint64_t n_proteins;              /* proteins kept by the FASTA parser */
    uint64_t n_windows, n_groups, n_candidates, n_rows;   /* length-filtered windows, group_digests groups, (group, combination) candidates, rows before the merge */
    uint64_t device_bytes;            /* HBM the handle holds (the output table) */
    uint64_t peak_device_bytes;       /* HBM the call held at its peak (temporaries and output) */
    float ms_parse;                   /* host wall clock of the FASTA parse and the parameter normalisation */
    float ms_upload, ms_sites, ms_windows, ms_group, ms_expand, ms_sort, ms_merge, ms_total;   /* CUDA-event stage times */
    float ms_wall;                    /* host wall clock of the create call */
} sage_b200_digest_info;

/* EINVAL for a null fasta (with fasta_len > 0), params or out, a null spec array with a nonzero count, or a non-finite mod mass; ELIMIT for
 * max_len > 255, max_variable_mods > 8, 2^32 or more residues, 2^32 - 2 or more windows, candidates or output rows, more than 65535
 * variable sites on one peptide, or when the work buffers do not fit the device's free memory (checked before each stage allocates; the
 * message names the byte count). An empty FASTA, or one whose every peptide is filtered, gives an empty table. */
int sage_b200_digest_create(int device, const char* fasta, uint64_t fasta_len, const sage_b200_digest_params* params, sage_b200_digest** out);
int sage_b200_digest_get_info(const sage_b200_digest* d, sage_b200_digest_info* info);
/* Any pointer may be NULL. residue_offsets / protein_offsets: [n_peptides + 1]; sequence / modifications: [n_residues]; nterm, cterm (NaN =
 * None), monoisotopic, decoy, missed_cleavages, semi_enzymatic: [n_peptides]; protein_ids: [n_protein_refs], ascending within a peptide, each
 * the rank of the accession in the names table (a repeated accession stays repeated); name_offsets: [n_names + 1] into name_bytes
 * [name_bytes]: the distinct accessions in byte order. */
int sage_b200_digest_export(const sage_b200_digest* d, uint32_t* residue_offsets, uint8_t* sequence, float* modifications, float* nterm, float* cterm,
                            float* monoisotopic, uint8_t* decoy, uint8_t* missed_cleavages, uint8_t* semi_enzymatic, uint32_t* protein_offsets,
                            uint32_t* protein_ids, uint64_t* name_offsets, char* name_bytes);
void sage_b200_digest_destroy(sage_b200_digest* d);

/* ---------------------------------------------------------------------------------------------------------------------------------------------
 * Prefilter (database.prefilter = true; runner.rs:104-128, 161-278): the FASTA's proteins are cut into consecutive chunks; each chunk is
 * digested and indexed, Scorer::quick_score (with report_psms + 1) runs every MS2 spectrum with at least min_peaks peaks against that index,
 * and only the peptides some spectrum selected are kept. The kept rows of all chunks are merged by reorder_peptides (database.rs:221-258)
 * and one final index is built from the merged table. Everything after the FASTA parse runs on the device and no table crosses PCIe. The
 * table is the reference's bit for bit under the definitions of DESIGN.md §15; protein ids are ranks in the names table of the whole FASTA.
 * create -> get_info -> export / chunk_counts / take_db -> destroy.
 */
typedef struct sage_b200_prefilter sage_b200_prefilter;

typedef struct {
    uint64_t chunk_size;              /* proteins per chunk; 0 = auto_calculate_prefilter_chunk_size (database.rs:142-160) */
    uint8_t low_memory;               /* prefilter_low_memory: the branch of quick_score (scoring.rs:270) */
    uint64_t min_peaks;               /* spectra with fewer peaks are not scored (runner.rs:255) */
} sage_b200_prefilter_params;

typedef struct {
    uint64_t chunk_size, n_chunks;    /* the chunk size used; chunks digested (0 with the plain build) */
    uint64_t plain_build;             /* 1: chunk_size >= the protein count, the plain digest was built and nothing was scored (runner.rs:110) */
    uint64_t n_proteins;              /* proteins kept by the FASTA parser (Fasta::targets) */
    uint64_t unmodified_peptides;     /* fasta.digest(&enzyme).len() when the chunk size was computed, else 0 */
    uint64_t n_spectra;               /* spectra scored against each chunk (MS2 with at least min_peaks peaks) */
    uint64_t rows_digested, rows_kept;/* peptides of the chunk tables, and those kept, over all chunks */
    uint64_t n_peptides, n_residues, n_protein_refs, n_names, name_bytes;   /* the export's array sizes */
    uint64_t n_fragments;             /* fragments of the final index */
    uint64_t device_bytes;            /* HBM the handle holds (the final table and, until taken, the final index) */
    uint64_t peak_device_bytes;       /* HBM the call held at its peak as counted by the library (the scorer's work buffers are not counted) */
    float ms_parse;                   /* host wall clock of the FASTA parse, the names table and the argument checks */
    float ms_count, ms_digest, ms_index, ms_quick_score, ms_compact, ms_merge, ms_final_index;   /* stage times summed over chunks: each stage
                                         ends with its work finished, so these are wall clock of device work (count: the automatic chunk size) */
    float ms_spectra_upload;          /* the part of ms_quick_score spent copying the spectra to the device (once per chunk) */
    float ms_wall;                    /* host wall clock of the create call */
} sage_b200_prefilter_info;

/* EINVAL (before the device is looked at) for a null required pointer, a null spec array with a nonzero count, a non-finite mod mass,
 * report_psms == 0, a bad tolerance kind or score type, bucket_size not a power of two, or bad ion kinds; ELIMIT for report_psms + 1 > 64 and
 * the digest's limits. EINVAL when the automatic chunk size is 0 (the reference panics in `chunks(0)`); ELIMIT when a stage's work buffers
 * do not fit the device's free memory (checked before it allocates). bucket_size, ion_kinds and min_ion_index are those of
 * sage_b200_db_build and serve every chunk index and the final index. */
int sage_b200_prefilter_create(int device, const char* fasta, uint64_t fasta_len, const sage_b200_digest_params* digest, const sage_b200_scorer_params* scorer,
                               const sage_b200_prefilter_params* params, const sage_b200_spectra* spectra, uint64_t bucket_size, const uint8_t* ion_kinds,
                               uint64_t n_ion_kinds, uint64_t min_ion_index, sage_b200_prefilter** out);
int sage_b200_prefilter_get_info(const sage_b200_prefilter* f, sage_b200_prefilter_info* info);
/* Per chunk, in chunk order: rows of its digest and rows kept ([n_chunks] each; either may be NULL). */
int sage_b200_prefilter_chunk_counts(const sage_b200_prefilter* f, uint64_t* rows_digested, uint64_t* rows_kept);
/* The final table, in the arrays and sizes of sage_b200_digest_export. */
int sage_b200_prefilter_export(const sage_b200_prefilter* f, uint32_t* residue_offsets, uint8_t* sequence, float* modifications, float* nterm, float* cterm,
                               float* monoisotopic, uint8_t* decoy, uint8_t* missed_cleavages, uint8_t* semi_enzymatic, uint32_t* protein_offsets,
                               uint32_t* protein_ids, uint64_t* name_offsets, char* name_bytes);
/* Hands the final index to the caller, who destroys it with sage_b200_db_destroy; EINVAL on a second call. */
int sage_b200_prefilter_take_db(sage_b200_prefilter* f, sage_b200_db** out);
void sage_b200_prefilter_destroy(sage_b200_prefilter* f);

/* ---------------------------------------------------------------------------------------------------------------------------------------------
 * Result files (runner.rs Runner::run, the CSV writers): the bytes of a Sage output file, formatted on the device as the reference writes
 * them (csv-core's tab-separated records, quoted only where a field holds '\t', '"', '\r' or '\n'; f32 / f64 in ryu's shortest round-trip
 * layout; integers as itoa; modification masses as Rust's `{:+}`). The definitions are DESIGN.md §17. One pass measures every record, a
 * scan places them, a second pass writes them chunk by chunk into at most text_budget bytes of device memory, and each chunk is copied once
 * to its offset in `out`.
 *   SAGE_B200_FILE_RESULTS    results.sage.tsv (runner.rs:687-780, 842-884): one record per row, in the caller's order
 *   SAGE_B200_FILE_PIN        results.sage.pin (runner.rs:938-1120): one record per row; log1p / log1pf are glibc's (the host libm's variant)
 *   SAGE_B200_FILE_FRAGMENTS  matched_fragments.sage.tsv (runner.rs:782-829, 904-936): one record per fragment of each row, rows in order,
 *                             fragments[rows[i].fragment_offset .. + fragment_count) in order
 *   SAGE_B200_FILE_LFQ        lfq.tsv (runner.rs:1182-1240): one record per target row of sage_b200_lfq_integrate, in its order (the
 *                             reference's order is a HashMap's: the set of records is the reference's, the order is defined here)
 *   SAGE_B200_FILE_TMT        tmt.tsv (runner.rs:1140-1180): one record per quantified spectrum in the caller's order
 * Strings the device does not own arrive as CSR byte tables: string i is bytes[offsets[i] .. offsets[i + 1]).
 */
#define SAGE_B200_FILE_RESULTS 1
#define SAGE_B200_FILE_PIN 2
#define SAGE_B200_FILE_FRAGMENTS 3
#define SAGE_B200_FILE_LFQ 4
#define SAGE_B200_FILE_TMT 5
typedef struct {
    float ms_upload, ms_measure, ms_scan, ms_write, ms_d2h, ms_total;   /* CUDA-event stage times (write and d2h summed over chunks) */
    uint64_t h2d_bytes, d2h_bytes, records, chunks;
} sage_b200_write_stats;
typedef struct {
    /* rows: results, pin, fragments */
    const sage_b200_feature* rows;        /* [n_rows] as the search returns them */
    const uint64_t* psm_id;               /* [n_rows] Feature::psm_id (the reference takes it from a global counter, so it is the caller's) */
    uint64_t n_rows;
    const sage_b200_fragment* fragments;  /* [n_fragments] as sage_b200_score_batch returns them with annotate_matches; kind 0..5 = a b c x y z */
    uint64_t n_fragments;
    /* strings: results, pin, tmt (filenames also lfq's header) */
    const uint64_t* filename_offsets;     /* [n_files + 1] */
    const char* filename_bytes;
    uint64_t n_files;
    const uint64_t* spec_id_offsets;      /* [n_spec_ids + 1] */
    const char* spec_id_bytes;
    uint64_t n_spec_ids;
    /* tmt.tsv */
    uint64_t n_quant;
    const uint32_t* quant_file_id;        /* [n_quant] < n_files */
    const uint32_t* quant_spec_id;        /* [n_quant] < n_spec_ids */
    const float* ion_injection_time;      /* [n_quant] */
    const float* peaks;                   /* [n_quant * n_channels] TmtQuant::peaks, row-major */
    uint64_t n_channels;
    uint8_t user_labels;                  /* 1: the columns are user_1..n (Isobaric::User), else tmt_1..n */
    /* the peptide table (results, pin, lfq): the digest's (sage_b200_digest_export) */
    const sage_b200_peptides* peptides;   /* residue_offsets, sequence, modifications, nterm and decoy are read */
    const float* cterm;                   /* [n_peptides] NaN = None; NULL = None for every peptide */
    const uint8_t* semi_enzymatic;        /* [n_peptides]; NULL = 0 */
    const uint32_t* protein_offsets;      /* [n_peptides + 1] */
    const uint32_t* protein_ids;          /* each < n_names */
    const uint64_t* name_offsets;         /* [n_names + 1] the protein names */
    const char* name_bytes;
    uint64_t n_names;
    const char* decoy_tag;                /* NULL = "rev_" */
    uint8_t generate_decoys;
    /* results / pin, per row: file and spectrum id, and the post-search columns, each [n_rows] or NULL for Feature's default
       (scoring.rs:575-592: aligned_rt = rt, predicted 0.0, deltas 0.999, discriminant 0.0, posterior_error and the q-values 1.0) */
    const uint32_t* file_id;              /* < n_files */
    const uint32_t* spec_index;           /* < n_spec_ids: the row's Feature::spec_id */
    const float *discriminant_score, *posterior_error, *spectrum_q;           /* sage_b200_spectrum_fdr */
    const float *aligned_rt, *predicted_rt, *delta_rt_model, *predicted_ims, *delta_ims_model;   /* sage_b200_predict_rt */
    const float *peptide_q, *protein_q;                                      /* sage_b200_picked_fdr */
    /* sage_b200_protein_groups' outputs (results): NULL group_pass = no groups (protein_groups empty). The string rule is the one stated
       above sage_b200_protein_groups; group ids < n_groups */
    const uint32_t* num_protein_groups;   /* [n_rows] or NULL = 0 */
    const float* protein_group_q;         /* [n_rows] or NULL = 1.0 */
    const uint8_t* group_pass;            /* [n_rows] */
    const uint64_t* row_group_offsets;    /* [n_rows + 1] */
    const uint32_t* row_groups;
    const uint64_t* group_offsets;        /* [n_groups + 1] */
    const uint32_t* group_members;        /* each < n_names */
    const uint8_t* group_decoy;           /* [n_groups] */
    uint64_t n_groups;
    /* lfq.tsv: sage_b200_lfq_integrate's rows and areas, sage_b200_picked_precursor's q-values */
    const sage_b200_lfq_row* lfq_rows;    /* [n_lfq] peptide < n_peptides */
    const double* lfq_areas;              /* [n_lfq * n_files] */
    const float* lfq_q;                   /* [n_lfq] */
    uint64_t n_lfq;
    uint64_t text_budget;                 /* device bytes of text per chunk; 0 = 256 MiB. A test hook: any value gives the same bytes (a chunk
                                             holds at least one block of 4096 records, so a block larger than the budget is one chunk) */
    sage_b200_write_stats* stats;         /* optional */
} sage_b200_write_inputs;
/* out == NULL: *bytes = the file's size, nothing written. Else: ELIMIT with *bytes set and nothing written when capacity < the size; else the
 * file is written to out[0 .. *bytes). EINVAL, before the device is looked at, for an unknown file, a null required pointer, a peptide_idx
 * outside the table, a file id >= n_files, a spectrum index >= n_spec_ids, a fragment range outside the fragment array, a fragment kind
 * outside 0..5, a protein id >= n_names, a group id >= n_groups or offsets that decrease (these checks read every input once); ELIMIT
 * beyond 2^32 - 1 records (or rows), or when the work buffers do not fit the device's free memory (checked before allocating; the
 * message names the byte count). A file with no records is its header alone and needs no device. */
int sage_b200_write_tsv(int device, int file, const sage_b200_write_inputs* in, char* out, uint64_t capacity, uint64_t* bytes);
/* Test hook: the per-block FNV-1a 64 hashes of formatted values, each followed by '\n'. format 0: ryu layout of the f32 with bits
 * first + i; 1: `{:+}` of the same f32; 2: ryu layout of the f64 values[i]. Block b covers values [b * block, (b + 1) * block) of n; hashes[n / block]
 * (n a multiple of block). */
int sage_b200_format_hashes(int device, int format, uint64_t first, const double* values, uint64_t n, uint64_t block, uint64_t* hashes);

/* Page-locked host buffers: spectra/feature arrays placed here are copied by DMA without a staging memcpy. */
void* sage_b200_host_alloc(size_t bytes);
/* The same for a batch sage_b200_score_batch_multi cuts into n_devices contiguous blocks: the i-th of n equal parts of the buffer is placed on the
 * NUMA node next to devices[i] (first touch by a bound thread), then the region is registered with CUDA. Release with sage_b200_host_free. */
void* sage_b200_host_alloc_blocks(size_t bytes, const int* devices, int n_devices);
void sage_b200_host_free(void* p);

/* Message of the last failure on the calling thread. Returns the message length. */
size_t sage_b200_last_error(char* buf, size_t cap);

/* ---------------------------------------------------------------------------------------------------------------------------------------------
 * MGF reader (MgfReader::parse, sage-cloudpath mgf.rs:324-370): the bytes of a whole MGF file -> its RawSpectrum list, parsed on the device
 * (DESIGN.md §18). The text must be UTF-8 (read_to_string); lines are `str::lines`, each `trim`med of Unicode White_Space; numbers are
 * `str::parse::<f32>`, correctly rounded. A record ends at a line starting "END IONS"; it is dropped when its id is empty, it has no
 * precursor, no peak, or more m/z than intensities. The first record does not see the header's TOL / TOLU / CHARGE (only QueryData::init
 * copies them in). create -> get_info -> export (caller-allocated arrays) and/or process -> destroy.
 */
typedef struct sage_b200_mgf sage_b200_mgf;
typedef struct {
    uint64_t n_bytes, n_lines, n_records;   /* the input; records: END IONS lines after the header */
    uint64_t n_spectra, n_peaks, n_precursors, id_bytes;   /* the export's array sizes */
    uint64_t dropped_records;               /* records check_spectrum rejected */
    uint64_t malformed_lines;               /* peak lines (led by an ASCII digit) whose m/z does not parse, PEPMASS= lines whose m/z does not */
    uint64_t file_id;
    uint64_t device_bytes;                  /* HBM the handle holds (the spectra) */
    uint64_t peak_device_bytes;             /* HBM the create call held at its peak */
    float ms_h2d, ms_read;                  /* CUDA-event times of the text's upload and of the parse that follows it */
} sage_b200_mgf_info;
/* EINVAL for a null out (or text with len > 0), invalid UTF-8 (the message names the first bad byte offset) or no line starting
 * "BEGIN IONS" (the reference panics); ELIMIT when a stage does not fit the device's free memory (the message names the byte count) or
 * past 2^31 - 16 records. */
int sage_b200_mgf_create(int device, const char* text, uint64_t len, uint64_t file_id, sage_b200_mgf** out);
int sage_b200_mgf_get_info(const sage_b200_mgf* m, sage_b200_mgf_info* info);
/* Any pointer may be NULL. peak_offsets, precursor_offsets, id_offsets: [n_spectra + 1]; mz, intensity: [n_peaks] in file order;
 * scan_start_time (RTINSECONDS / 60, else 0) and tic (the f32 sum of the intensities in file order): [n_spectra]. Precursors, [n_precursors]:
 * every PEPMASS x every charge of the CHARGE list, in that nesting; intensity with its Some flag; charge with its Some flag (Some(0) is a
 * value); isolation_kind 0 = None, 1 = Da, 2 = ppm with (isolation_lo, isolation_hi) = (-|TOL|, |TOL|). id_bytes: [id_bytes], the TITLEs. */
int sage_b200_mgf_export(const sage_b200_mgf* m, uint64_t* peak_offsets, float* mz, float* intensity, float* scan_start_time, float* tic,
                         uint64_t* precursor_offsets, float* precursor_mz, float* precursor_intensity, uint8_t* precursor_intensity_some,
                         uint8_t* precursor_charge, uint8_t* precursor_charge_some, uint8_t* isolation_kind, float* isolation_lo,
                         float* isolation_hi, uint64_t* id_offsets, char* id_bytes);
/* SpectrumProcessor::process (level 2, as sage_b200_process_spectra) of the handle's spectra where they are on the device. Each spectrum's
 * charge is its first precursor's (None -> 0, which the processor takes as unwrap_or(3)). ELIMIT when a first precursor's charge is
 * Some(0) (the message names the spectrum), past the processor's shared-memory budget, or past 2^31 - 1 spectra or 2^32 - 16 peaks.
 * out_offsets[n_spectra + 1]; out_masses / out_intensities sized for n_peaks; out_tic[n_spectra]. */
int sage_b200_mgf_process(const sage_b200_mgf* m, const sage_b200_processor_params* processor, uint64_t* out_offsets, float* out_masses,
                          float* out_intensities, float* out_tic);
void sage_b200_mgf_destroy(sage_b200_mgf* m);
/* Test hook: out[i], ok[i] = str::parse::<f32> of bytes[offsets[i] .. offsets[i+1]) on the device (ok 0: an Err; out is then 0). EINVAL for
 * null arrays or decreasing offsets, before any device call. */
int sage_b200_parse_f32(int device, const char* bytes, const uint64_t* offsets, uint64_t n, float* out, uint8_t* ok);

#ifdef __cplusplus
}
#endif
#endif /* SAGE_B200_H */
