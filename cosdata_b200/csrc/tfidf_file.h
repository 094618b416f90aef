// tfidf_file.h -- the reference's TF-IDF index files (tf_idf_index/index-tree.dim and <version>.idat) as read by
// tfidf_file.cu: the state TFIDFIndexRoot::deserialize rebuilds, kept as the list records themselves so that
// cdb_tfidf_index_load_files (tfidf.cu) can upload them unchanged.  Host-only.
#pragma once
#include <map>
#include <memory>
#include <vector>

#include "ref_files.h"

// one record of a term's chain as deserialize keeps it: its `len` words start at byte `words` of file `file`
struct TfIdfFileRecord {
    const uint8_t *words;   // inside the mapping of `<version>.idat`
    uint64_t base;          // position of its first word in the concatenation of every kept record, in term and chain order
    uint32_t len;
    uint32_t term;          // index into cdb_tfidf_files::hashes
    uint32_t version;
};

struct cdb_tfidf_files {
    uint32_t n_docs = 0;                                             // total_documents_count
    std::map<uint32_t, std::unique_ptr<cdb::reffiles::Mapped>> idat; // by version
    std::unique_ptr<cdb::reffiles::Mapped> dim;
    std::vector<uint32_t> hashes, df;                                // ascending hashes; df = VersionedVec::len
    std::vector<uint64_t> rec_begin;                                 // term t's records are recs[rec_begin[t] .. rec_begin[t + 1])
    std::vector<TfIdfFileRecord> recs;
    std::vector<uint64_t> killed;                                    // ascending positions (as TfIdfFileRecord::base) deserialize marks u64::MAX
    uint64_t n_words = 0, n_live = 0, max_id_end = 0;                // words in the kept records, live words, largest live id + 1
    uint32_t max_version = 0;                                        // largest version of a kept record
};
