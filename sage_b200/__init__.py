"""sage_b200 — H100-native (sm_90a) fragment-index search-and-score, a drop-in for sage-core's
`IndexedDatabase::query` + `Scorer::score` hot path (lazear/sage). The product is the CUDA library behind the C ABI
in include/sage_b200.h; this package is the thin Python binding used by the tests and the benchmark."""
from .api import (DA, PCT, PPM, Feature, IndexedDatabase, Peptides, Precursor, ProcessedSpectrum, Scorer, SpectraBatch, SpectrumProcessor, Tolerance,  # noqa: F401
                  SageB200Error, device_count, FeatureMap, LfqSettings, Ms1Batch, spectrum_fdr, predict_rt, picked_fdr, picked_precursor,
                  competition_keys, protein_groups, protein_group_strings, bipartite_cover,
                  DigestResult, digest_fasta, PrefilterResult, prefilter_fasta, RawSpectra, ProcessedBatch, ISOBARIC, tmt_quantify,
                  tmt_min_deisotope_mz, MgfSpectra, read_mgf)
from .build import build_library, library_path  # noqa: F401
