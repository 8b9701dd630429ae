"""rucene_b200 — H100-native query evaluation for Rucene's IndexSearcher hot path.

Layout (only what the path needs):
  csrc/gpu/    hand-written sm_90a CUDA kernels + the C ABI (include/rucene_gpu.h)
  csrc/codec/  host write side of the Lucene50 postings format + synthetic index generator
  csrc/host/   C++ mirror of the reference's Query/Weight/Collector surface over the C ABI
  engine.py    ctypes binding of librucene_gpu.so (fails loudly when CUDA is unavailable)
  search.py    Python mirror of IndexSearcher/TermQuery/BooleanQuery/TopDocsCollector
"""
__version__ = "0.1.0"
