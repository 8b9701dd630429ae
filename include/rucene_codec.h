/*
 * rucene_codec.h — host-side C ABI (librucene_codec.so): the write side of the Lucene50
 * postings format for a DocsAndFreqs field, the BM25 weight computation the Query/Weight layer
 * performs once per query, and the synthetic index generator used by tests and bench.py.
 *
 * This is the "data format either side of the path": it produces real `.doc` byte streams
 * (IndexHeader + ForUtil table + per-term block/vint/skip regions + footer) that both the
 * CPU reference algorithm and the GPU engine consume.  Reference interfaces are cited per
 * function; paths are relative to src/core/ of zhihu/rucene.
 */
#ifndef RUCENE_CODEC_H
#define RUCENE_CODEC_H
#include <stddef.h>
#include <stdint.h>

#include "rucene_gpu.h" /* rg_term_state */

#ifdef __cplusplus
extern "C" {
#endif

typedef struct rc_writer rc_writer;
typedef struct rc_segment rc_segment;
typedef struct rc_blocks rc_blocks;

const char* rc_last_error(void);

/* ---- Lucene50PostingsWriter for one DocsAndFreqs field (codec/postings/posting_writer.rs) --
 * doc_version 1: Rucene's SIMD128 block layout (what the reference writes, :201-205);
 * doc_version 0: stock Lucene 5/6 layout (Packed / PackedSingleBlock per the COMPACT table). */
rc_writer* rc_writer_create(int doc_version, int32_t max_doc, const uint8_t segment_id[16],
                            const char* suffix);
/* start_term / start_doc / finish_doc / finish_term (:289-361, :457-474, :477-589) for one term
 * whose postings are docs[0..n) strictly ascending with freqs[i] >= 1. */
int rc_writer_add_term(rc_writer* w, const int32_t* docs, const int32_t* freqs, int32_t n,
                       rg_term_state* out_state);
/* Turn on the reference's dormant doc-block encodings for the terms added afterwards
 * (EfWriterMeta{use_ef, with_pf}, codec/postings/posting_writer.rs:33-57; ForUtil::write_block,
 * for_util.rs:417-468): a block whose 128 docids fit a FixedBitSet no larger than its PF payload is
 * written as EncodeType::BITSET, else as EncodeType::EF (Elias-Fano) when that is no larger than PF
 * (or always, with_pf = 0), else as PF.  The open-source writer never sets use_ef; production
 * indexes carry these blocks and the reader side handles them (posting_reader.rs:501-561). */
int rc_writer_set_ef(rc_writer* w, int use_ef, int with_pf);
/* EliasFanoEncoder pieces, exported so the reference's own unit vectors can be checked
 * (util/packed/elias_fano_encoder.rs:308-311 num_longs_for_bits, :334-345 pack_value, :46-253
 * new + encode_next: out_longs = upper | lower | index longs, out_geom = {num_low_bits, n_upper,
 * n_lower, n_index}). */
int64_t rc_ef_num_longs_for_bits(int64_t n);
void rc_ef_pack_value(int64_t value, int64_t* longs, int n_longs, int num_bits, int64_t pack_index);
int rc_ef_encode(const int64_t* values, int64_t n, int64_t upper_bound, int64_t* out_longs, int cap,
                 int32_t out_geom[4]);
/* out[0] full blocks written, out[1] of them EF, out[2] of them BITSET */
void rc_writer_block_counts(rc_writer* w, uint64_t out[3]);
int rc_writer_finish(rc_writer* w); /* codec footer (codec/codec_util.rs:110-114) */
const uint8_t* rc_writer_data(rc_writer* w, size_t* len);
/* the 32 ForUtil header codes as written (codec/postings/for_util.rs:150-185) */
void rc_writer_forutil_table(rc_writer* w, int32_t out[32]);
void rc_writer_destroy(rc_writer* w);

/* ForUtil::write_block (for_util.rs:396-478) for one 128-value block appended to `out`
 * (capacity >= 1+512).  Returns bytes written. */
int rc_forutil_write_block(const int32_t data[128], int doc_version, uint8_t* out);

/* ---- BM25 host side (search/similarity/bm25_similarity.rs, util/small_float.rs) ---- */
uint8_t rc_float_to_byte315(float f);
float rc_byte315_to_float(uint8_t b);
uint8_t rc_encode_norm_value(float boost, int32_t field_length); /* :90-92 */
float rc_bm25_idf(int64_t doc_freq, int64_t doc_count);          /* :99-114 */
float rc_bm25_avg_field_length(int64_t sum_total_term_freq, int64_t doc_count, int64_t max_doc); /* :72-83 */
void rc_bm25_norm_cache(float k1, float b, float avgdl, float out_cache[256]); /* :161-165 */

/* ---- synthetic Zipfian segment (SURVEY.md §8d) -------------------------------------- */
typedef struct {
    uint64_t seed;
    int32_t max_doc;     /* N */
    uint32_t n_terms;    /* V; term id t has rank r=t+1, target df = max(1, N/(r+1)) */
    int32_t doc_version; /* 0 | 1 */
    int32_t n_threads;   /* <=0: all hardware threads */
} rc_synth_config;

rc_segment* rc_synth_segment(const rc_synth_config* cfg);
void rc_segment_destroy(rc_segment* s);
const uint8_t* rc_segment_doc_file(const rc_segment* s, size_t* len);
const uint8_t* rc_segment_norms(const rc_segment* s);             /* max_doc bytes */
const rg_term_state* rc_segment_terms(const rc_segment* s, uint32_t* n_terms);
/* out[0]=doc_count, [1]=sum_total_term_freq, [2]=sum_doc_freq, [3]=max_doc, [4]=total full
 * blocks, [5]=total postings */
void rc_segment_stats(const rc_segment* s, int64_t out[8]);
void rc_segment_forutil_table(const rc_segment* s, int32_t out[32]);

/* ---- synthetic block stream for the ForUtil microbench (BASELINE config 2) ---------
 * mode 0: uniform widths b in [1,32], values uniform in [0,2^b) with one forced top bit;
 * mode 1: fixed width `param` (0 = all-equal blocks) ; returns stream + offsets. */
rc_blocks* rc_synth_blocks(uint64_t seed, uint32_t n_blocks, int mode, int param,
                           int doc_version);
const uint8_t* rc_blocks_stream(const rc_blocks* b, size_t* len);
const uint64_t* rc_blocks_offsets(const rc_blocks* b, uint32_t* n);
/* the raw values the blocks encode (n_blocks*128), for round-trip checks */
const int32_t* rc_blocks_values(const rc_blocks* b);
void rc_blocks_forutil_table(int32_t out[32]);
void rc_blocks_destroy(rc_blocks* b);

int rc_hardware_threads(void);

#ifdef __cplusplus
}
#endif
#endif
