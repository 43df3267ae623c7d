"""
cutadapt_b200 -- H100-native adapter-trimming core with cutadapt's adapter/aligner API.

The package mirrors the *hot path* of marcelm/cutadapt and nothing else:

    cutadapt_b200._align          Aligner, PrefixComparer, SuffixComparer, hamming_sphere,
                                  edit_environment              (ref: src/cutadapt/_align.pyx)
    cutadapt_b200.align           EndSkip + re-exports          (ref: src/cutadapt/align.py)
    cutadapt_b200._kmer_finder    KmerFinder                    (ref: src/cutadapt/_kmer_finder.pyx)
    cutadapt_b200.kmer_heuristic  create_positions_and_kmers    (ref: src/cutadapt/kmer_heuristic.py)
    cutadapt_b200.qualtrim        quality_trim_index            (ref: src/cutadapt/qualtrim.pyx)
    cutadapt_b200.adapters        the Adapter classes, Match classes, MultipleAdapters
                                                                (ref: src/cutadapt/adapters.py)
    cutadapt_b200.pipeline        batched per-chunk dispatch    (ref: pipeline.py + modifiers.py
                                                                 AdapterCutter/QualityTrimmer)

All per-read work runs in hand-written sm_90a CUDA kernels behind the C ABI declared in
include/cutadapt_b200.h (cutadapt_b200/libcutadapt_b200.so, loaded with ctypes).  There is no
CPU fallback: without the built library and a CUDA device the first call raises.
"""
__version__ = "0.1.0"
__all__ = ["__version__"]
