// qdrant_b200.hpp — C++ host side above the C ABI (include/qb200.h), mirroring the reference's scorer interface.
//
// The reference is compiled (Rust) code and its toolchain is absent from the build image, so the host-side mirror of
// its operator interface is written in C++ (header only; links against libqdrant_b200.so):
//     RawScorer               lib/segment/src/vector_storage/raw_scorer.rs:39-54
//     RawScorerBuilder        raw_scorer.rs:122-128
//     FilteredScorer          lib/segment/src/index/hnsw_index/point_scorer.rs:53-58,160-304
//     BatchFilteredSearcher   point_scorer.rs:312-472
//     ScoredPointOffset       lib/common/common/src/types.rs:12-31
//     GraphLayers::search     lib/segment/src/index/hnsw_index/graph_layers.rs:530-561   (HnswGraph: whole batches on the device)
//     SegmentsSearcher task + BatchResultAggregator   segments_searcher.rs:255, search_result_aggregator.rs:50-117   (SegmentShard)
// Same names, argument meaning and error behaviour: construction may fail (OperationError -> std::runtime_error),
// scoring is infallible apart from device failures (which throw, the analogue of the reference's `expect`).
#pragma once
#include <algorithm>
#include <atomic>
#include <cstdint>
#include <functional>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/qb200.h"

namespace qdrant_b200 {

using PointOffsetType = uint32_t;  // common::types::PointOffsetType
using ScoreType = float;           // common::types::ScoreType
using ScoredPointOffset = qb_scored_point;
constexpr size_t VECTOR_READ_BATCH_SIZE = 64;  // vector_storage/common.rs:20

struct OperationError : std::runtime_error {
    qb_status status;
    OperationError(qb_status s, const std::string& what) : std::runtime_error(what), status(s) {}
};
inline void check(qb_status st) {
    if (st != QB_OK) throw OperationError(st, qb_last_error());
}

enum class Distance : int { Cosine = QB_DIST_COSINE, Euclid = QB_DIST_EUCLID, Dot = QB_DIST_DOT, Manhattan = QB_DIST_MANHATTAN };

// Box<dyn RawScorer + 'a>
class RawScorer {
public:
    virtual ~RawScorer() = default;
    virtual void score_points(const PointOffsetType* points, size_t n, ScoreType* scores) const = 0;
    virtual ScoreType score_point(PointOffsetType point) const = 0;
    virtual ScoreType score_internal(PointOffsetType a, PointOffsetType b) const = 0;
};

class VectorStorage;

class B200RawScorer final : public RawScorer {
public:
    B200RawScorer(qb_scorer* h) : h_(h) {}
    ~B200RawScorer() override { qb_scorer_destroy(h_); }
    B200RawScorer(const B200RawScorer&) = delete;
    void score_points(const PointOffsetType* points, size_t n, ScoreType* scores) const override { check(qb_score_points(h_, points, n, scores)); }
    ScoreType score_point(PointOffsetType point) const override {
        ScoreType s;
        check(qb_score_point(h_, point, &s));
        return s;
    }
    ScoreType score_internal(PointOffsetType a, PointOffsetType b) const override {
        ScoreType s;
        check(qb_score_internal(h_, a, b, &s));
        return s;
    }
    qb_scorer* raw() const { return h_; }

private:
    qb_scorer* h_;
};

// A segment's vectors resident in HBM; doubles as RawScorerBuilder / QuantizedVectorsRead.
class VectorStorage {
public:
    explicit VectorStorage(qb_storage* h) : h_(h) {}
    ~VectorStorage() { qb_storage_destroy(h_); }
    VectorStorage(const VectorStorage&) = delete;

    static std::unique_ptr<VectorStorage> dense_f32(int device, Distance d, uint32_t dim, uint64_t count, const float* rows) {
        qb_storage* h = nullptr;
        check(qb_storage_create_dense(device, QB_DT_F32, static_cast<qb_distance>(d), dim, count, rows, (uint64_t)dim * 4, &h));
        return std::make_unique<VectorStorage>(h);
    }
    static std::unique_ptr<VectorStorage> sq8(int device, Distance d, uint32_t dim, uint64_t count, const uint8_t* rows, uint32_t row_bytes, float alpha,
                                             float offset, float multiplier) {
        // construct_vector_parameters (quantized_vectors.rs:205-234)
        const qb_qdistance dt = (d == Distance::Euclid) ? QB_QD_L2 : (d == Distance::Manhattan ? QB_QD_L1 : QB_QD_DOT);
        const int invert = (d == Distance::Euclid || d == Distance::Manhattan) ? 1 : 0;
        qb_storage* h = nullptr;
        check(qb_storage_create_sq8(device, dim, count, rows, row_bytes, alpha, offset, multiplier, dt, invert, static_cast<qb_distance>(d), &h));
        return std::make_unique<VectorStorage>(h);
    }
    // RawScorerBuilder::build_raw_scorer / QuantizedVectorsRead::raw_scorer
    std::unique_ptr<RawScorer> build_raw_scorer(const float* query) const {
        qb_scorer* sc = nullptr;
        check(qb_scorer_create(h_, query, &sc));
        return std::make_unique<B200RawScorer>(sc);
    }
    // new_raw_scorer for QueryVector::{RecommendBestScore, RecommendSumScores, Discover, Context} (raw_scorer.rs:228-333):
    // `vectors` = the flattened example vectors in the layout include/qb200.h documents
    std::unique_ptr<RawScorer> build_custom_scorer(qb_query_kind kind, const float* vectors, uint32_t n_a, uint32_t n_b) const {
        qb_scorer* sc = nullptr;
        check(qb_scorer_create_custom(h_, kind, vectors, n_a, n_b, &sc));
        return std::make_unique<B200RawScorer>(sc);
    }
    // QuantizedVectorsRead::raw_internal_scorer (throws OperationError{QB_ERR_UNSUPPORTED} for PQ)
    std::unique_ptr<RawScorer> raw_internal_scorer(PointOffsetType point) const {
        qb_scorer* sc = nullptr;
        check(qb_scorer_create_internal(h_, point, &sc));
        return std::make_unique<B200RawScorer>(sc);
    }
    // mmr_from_points_with_vector (shard/src/query/mmr/mod.rs:42-279) over candidates whose vectors are this storage's rows: one query of
    // dim raw f32, (id, score) candidates in the storage's numbering, lambda = 1 - diversity -> the selection, with the input scores
    std::vector<qb_scored_point> mmr(const float* query, const std::vector<qb_scored_point>& candidates, float lambda, uint32_t limit,
                                     qb_hw_counters* counters = nullptr) const {
        std::vector<qb_scored_point> out(std::max<uint32_t>(limit, 1));
        const uint32_t n = (uint32_t)candidates.size();
        uint32_t count = 0;
        check(qb_mmr_batch(h_, query, 1, &lambda, candidates.data(), &n, n, limit, out.data(), &count, counters));
        out.resize(count);
        return out;
    }
    // the same over multivector candidates whose token rows are this storage's rows (point p = rows [point_offsets[p], point_offsets[p+1])):
    // one query of n_query_vectors x dim raw f32, (point offset, score) candidates, pair scores MaxSim -> the selection, with the input scores
    std::vector<qb_scored_point> mmr_maxsim(const std::vector<uint32_t>& point_offsets, const float* query_vectors, uint32_t n_query_vectors,
                                            const std::vector<qb_scored_point>& candidates, float lambda, uint32_t limit,
                                            qb_hw_counters* counters = nullptr) const {
        std::vector<qb_scored_point> out(std::max<uint32_t>(limit, 1));
        const uint32_t n = (uint32_t)candidates.size(), q_off[2] = {0, n_query_vectors};
        const uint32_t n_points = point_offsets.empty() ? 0 : (uint32_t)point_offsets.size() - 1;
        uint32_t count = 0;
        check(qb_mmr_maxsim_batch(h_, point_offsets.data(), n_points, query_vectors, q_off, 1, &lambda, candidates.data(), &n, n, limit, out.data(), &count,
                                  counters));
        out.resize(count);
        return out;
    }
    uint64_t count() const {
        uint64_t c = 0;
        check(qb_storage_info(h_, nullptr, &c, nullptr));
        return c;
    }
    uint32_t dim() const {
        uint32_t d = 0;
        check(qb_storage_info(h_, &d, nullptr, nullptr));
        return d;
    }
    qb_storage* raw() const { return h_; }

private:
    qb_storage* h_;
};

// point_scorer.rs:53-58: RawScorer + filters (deleted bitslice, optional payload filter)
class FilteredScorer {
public:
    FilteredScorer(std::unique_ptr<RawScorer> raw, const std::vector<bool>* point_deleted = nullptr,
                   std::function<bool(PointOffsetType)> filter = nullptr)
        : raw_(std::move(raw)), deleted_(point_deleted), filter_(std::move(filter)) {}

    bool check_vector(PointOffsetType p) const {
        if (deleted_ && p < deleted_->size() && (*deleted_)[p]) return false;
        return !filter_ || filter_(p);
    }
    // point_scorer.rs:265-295: filters `point_ids` in place, truncates to `limit` (0 = no limit), scores in ONE batch call
    std::vector<ScoredPointOffset> score_points(std::vector<PointOffsetType>& point_ids, size_t limit) {
        size_t kept = 0;
        for (PointOffsetType p : point_ids)
            if (check_vector(p)) point_ids[kept++] = p;
        point_ids.resize(kept);
        if (limit != 0 && point_ids.size() > limit) point_ids.resize(limit);
        scores_.resize(point_ids.size());
        raw_->score_points(point_ids.data(), point_ids.size(), scores_.data());
        std::vector<ScoredPointOffset> out(point_ids.size());
        for (size_t i = 0; i < point_ids.size(); ++i) out[i] = ScoredPointOffset{point_ids[i], scores_[i]};
        return out;
    }
    ScoreType score_point(PointOffsetType p) const { return raw_->score_point(p); }
    ScoreType score_internal(PointOffsetType a, PointOffsetType b) const { return raw_->score_internal(a, b); }

private:
    std::unique_ptr<RawScorer> raw_;
    const std::vector<bool>* deleted_;
    std::function<bool(PointOffsetType)> filter_;
    std::vector<ScoreType> scores_;
};

// point_scorer.rs:312-472: the reference walks 64-id chunks x per-query scorers x per-query heaps; here the scan and the
// top-k are one fused library call.
class BatchFilteredSearcher {
public:
    BatchFilteredSearcher(const float* queries, uint32_t n_queries, const VectorStorage& storage, uint32_t top, const uint64_t* point_deleted_words = nullptr)
        : queries_(queries), nq_(n_queries), st_(storage), top_(top), deleted_(point_deleted_words) {
        if (top == 0) throw std::invalid_argument("length must be greater than zero");  // FixedLengthPriorityQueue::new
    }
    // peek_top_all: every non-deleted point; is_stopped mirrors &AtomicBool (check_process_stopped)
    std::vector<std::vector<ScoredPointOffset>> peek_top_all(const std::atomic<int32_t>* is_stopped = nullptr) const { return run(nullptr, 0, is_stopped); }
    // peek_top_iter over an explicit id list (deferred / filtered points already removed by the caller)
    std::vector<std::vector<ScoredPointOffset>> peek_top_iter(const std::vector<PointOffsetType>& points, const std::atomic<int32_t>* is_stopped = nullptr) const {
        return run(points.data(), points.size(), is_stopped);
    }

private:
    std::vector<std::vector<ScoredPointOffset>> run(const PointOffsetType* ids, uint64_t n_ids, const std::atomic<int32_t>* is_stopped) const {
        std::vector<ScoredPointOffset> flat((size_t)nq_ * top_);
        std::vector<uint32_t> counts(nq_);
        static const PointOffsetType kNone = 0;
        check(qb_search_batch(st_.raw(), queries_, nq_, top_, deleted_, (ids || n_ids) ? (ids ? ids : &kNone) : nullptr, n_ids,
                              reinterpret_cast<const volatile int32_t*>(is_stopped), flat.data(), counts.data(), nullptr));
        std::vector<std::vector<ScoredPointOffset>> out(nq_);
        for (uint32_t q = 0; q < nq_; ++q) out[q].assign(flat.begin() + (size_t)q * top_, flat.begin() + (size_t)q * top_ + counts[q]);
        return out;
    }
    const float* queries_;
    uint32_t nq_;
    const VectorStorage& st_;
    uint32_t top_;
    const uint64_t* deleted_;
};

// GraphLayers::search (index/hnsw_index/graph_layers.rs:530-561) for a batch of queries, traversal and scoring on the device.
// The graph is the segment's links.bin in GraphLinksFormat::Plain (graph_links/view.rs:121-135) or, through compressed(),
// in GraphLinksFormat::Compressed (view.rs:137-163), the format the reference writes for every index it builds.
class HnswGraph {
public:
    HnswGraph(const VectorStorage& storage, const uint8_t* links_bin, uint64_t n_bytes, uint32_t m, uint32_t m0) {
        check(qb_hnsw_create_plain(storage.raw(), links_bin, n_bytes, m, m0, &h_));
    }
    // m and m0 are read from the compressed file's header
    static std::unique_ptr<HnswGraph> compressed(const VectorStorage& storage, const uint8_t* links_bin, uint64_t n_bytes) {
        qb_hnsw* h = nullptr;
        check(qb_hnsw_create_compressed(storage.raw(), links_bin, n_bytes, &h));
        return std::unique_ptr<HnswGraph>(new HnswGraph(h));
    }
    // a CompressedWithVectors links.bin (inline storage) bound to the segment's SQ8 storage (qb_hnsw_create_with_vectors)
    static std::unique_ptr<HnswGraph> with_vectors(const VectorStorage& quantized, const uint8_t* links_bin, uint64_t n_bytes) {
        qb_hnsw* h = nullptr;
        check(qb_hnsw_create_with_vectors(quantized.raw(), links_bin, n_bytes, &h));
        return std::unique_ptr<HnswGraph>(new HnswGraph(h));
    }
    // builds the graph of a dense f32 or Uint8 storage on the device (qb_hnsw_build); levels: one per point, <= 30; batch / serial_points 0 = 512 / 256.
    // The entry point the search starts from is returned in entry_point / entry_level.
    static std::unique_ptr<HnswGraph> build(const VectorStorage& storage, uint32_t m, uint32_t m0, uint32_t ef_construct, const std::vector<uint8_t>& levels,
                                            uint32_t batch, uint32_t serial_points, uint32_t& entry_point, uint32_t& entry_level) {
        qb_hnsw* h = nullptr;
        check(qb_hnsw_build(storage.raw(), m, m0, ef_construct, levels.data(), batch, serial_points, &h, &entry_point, &entry_level));
        return std::unique_ptr<HnswGraph>(new HnswGraph(h));
    }
    // builds the graph of a dense f32 or Uint8 storage from an old segment's graph of the same datatype (qb_hnsw_build_incremental): heals the old graph where points
    // have gone, renumbers it by old_to_new (one per old point; 0xFFFFFFFF = not carried over) and inserts only the new points.  levels:
    // one per point of `storage`, a mapped point's equal to its old level; m / m0 are old's; batch / serial_points 0 = 512 / 256.
    static std::unique_ptr<HnswGraph> build_incremental(const VectorStorage& storage, const HnswGraph& old, const std::vector<uint32_t>& old_to_new,
                                                        uint32_t ef_construct, const std::vector<uint8_t>& levels, uint32_t batch, uint32_t serial_points,
                                                        uint32_t& entry_point, uint32_t& entry_level) {
        qb_hnsw* h = nullptr;
        check(qb_hnsw_build_incremental(storage.raw(), old.h_, old_to_new.data(), ef_construct, levels.data(), batch, serial_points, &h, &entry_point,
                                        &entry_level));
        return std::unique_ptr<HnswGraph>(new HnswGraph(h));
    }
    // builds the graph over the points of a multivector collection on the device (qb_hnsw_build_multivector): point p = token rows
    // [point_offsets[p], point_offsets[p+1]) of the dense f32 `tokens`; levels: one per point; deleted_points: optional bitmap over points
    // (ceil(n / 64) words, may be null).  Search it with the MaxSim search.
    static std::unique_ptr<HnswGraph> build_multivector(const VectorStorage& tokens, const std::vector<uint32_t>& point_offsets, uint32_t m, uint32_t m0,
                                                        uint32_t ef_construct, const std::vector<uint8_t>& levels, const uint64_t* deleted_points,
                                                        uint32_t batch, uint32_t serial_points, uint32_t& entry_point, uint32_t& entry_level) {
        if (point_offsets.empty() || levels.size() + 1 != point_offsets.size()) throw OperationError(QB_ERR_INVALID, "levels and point_offsets disagree on the point count");
        qb_hnsw* h = nullptr;
        check(qb_hnsw_build_multivector(tokens.raw(), point_offsets.data(), (uint32_t)levels.size(), m, m0, ef_construct, levels.data(), deleted_points, batch,
                                        serial_points, &h, &entry_point, &entry_level));
        return std::unique_ptr<HnswGraph>(new HnswGraph(h));
    }
    // the graph as a plain links.bin (qb_hnsw_export_plain)
    std::vector<uint8_t> export_plain() const {
        uint64_t n = 0;
        check(qb_hnsw_export_plain(h_, nullptr, 0, &n));
        std::vector<uint8_t> out(n);
        check(qb_hnsw_export_plain(h_, out.data(), n, &n));
        return out;
    }
    ~HnswGraph() { qb_hnsw_destroy(h_); }
    HnswGraph(const HnswGraph&) = delete;
    // GraphLinks::links (view.rs:238-263): the point's links on `level`, in stored order
    std::vector<PointOffsetType> links(PointOffsetType point, uint32_t level) const {
        uint32_t count = 0;
        check(qb_hnsw_links(h_, level, &point, 1, 0, nullptr, &count));
        std::vector<PointOffsetType> out(count);
        if (count) check(qb_hnsw_links(h_, level, &point, 1, count, out.data(), &count));
        return out;
    }
    // SearchAlgorithm (graph_layers.rs:80-84): the level-0 algorithm; the caller decides as hnsw/read_view/search.rs:59-86 does
    enum class SearchAlgorithm : int32_t { Hnsw = QB_HNSW_ALGO_HNSW, Acorn = QB_HNSW_ALGO_ACORN };
    // entry_point / entry_level = GraphLayers::get_entry_point(filters, custom_entry_points); deleted = the filter as a bitmap (bit = 1: skip)
    std::vector<std::vector<ScoredPointOffset>> search(const float* queries, uint32_t n_queries, uint32_t top, uint32_t ef, PointOffsetType entry_point,
                                                       uint32_t entry_level, const uint64_t* deleted = nullptr,
                                                       SearchAlgorithm algorithm = SearchAlgorithm::Hnsw) const {
        std::vector<ScoredPointOffset> flat((size_t)n_queries * top);
        std::vector<uint32_t> counts(n_queries);
        check(qb_hnsw_search_batch_algo(h_, queries, n_queries, top, ef, entry_point, entry_level, deleted, nullptr, flat.data(), counts.data(), nullptr,
                                        static_cast<qb_hnsw_algorithm>(algorithm)));
        std::vector<std::vector<ScoredPointOffset>> out(n_queries);
        for (uint32_t q = 0; q < n_queries; ++q) out[q].assign(flat.begin() + (size_t)q * top, flat.begin() + (size_t)q * top + counts[q]);
        return out;
    }
    // GraphLayers::search_with_vectors on a with_vectors() graph (qb_hnsw_search_with_vectors_batch); ef = max(ef, oversampled top)
    std::vector<std::vector<ScoredPointOffset>> search_with_vectors(const float* queries, uint32_t n_queries, uint32_t top, uint32_t ef,
                                                                    PointOffsetType entry_point, uint32_t entry_level, const uint64_t* deleted = nullptr) const {
        std::vector<ScoredPointOffset> flat((size_t)n_queries * top);
        std::vector<uint32_t> counts(n_queries);
        check(qb_hnsw_search_with_vectors_batch(h_, queries, n_queries, top, ef, entry_point, entry_level, deleted, nullptr, flat.data(), counts.data(),
                                                nullptr));
        std::vector<std::vector<ScoredPointOffset>> out(n_queries);
        for (uint32_t q = 0; q < n_queries; ++q) out[q].assign(flat.begin() + (size_t)q * top, flat.begin() + (size_t)q * top + counts[q]);
        return out;
    }
    // custom queries (search.rs:181-208): vectors = n_queries x E x dim in the build_custom_scorer layout; coef = n_queries x (1 + n_a) for
    // feedback, else null; custom_entry_points = n_queries x n_custom ids, custom_counts[q] valid (or null)
    std::vector<std::vector<ScoredPointOffset>> search_custom(qb_query_kind kind, const float* vectors, uint32_t n_a, uint32_t n_b, const float* coef,
                                                              uint32_t n_queries, uint32_t top, uint32_t ef, PointOffsetType entry_point, uint32_t entry_level,
                                                              const uint32_t* custom_entry_points = nullptr, const uint32_t* custom_counts = nullptr,
                                                              uint32_t n_custom = 0, const uint64_t* deleted = nullptr,
                                                              SearchAlgorithm algorithm = SearchAlgorithm::Hnsw) const {
        std::vector<ScoredPointOffset> flat((size_t)n_queries * top);
        std::vector<uint32_t> counts(n_queries);
        check(qb_hnsw_search_custom_batch(h_, kind, vectors, n_a, n_b, coef, n_queries, top, ef, entry_point, entry_level, custom_entry_points, custom_counts,
                                          n_custom, deleted, nullptr, flat.data(), counts.data(), nullptr, static_cast<qb_hnsw_algorithm>(algorithm)));
        return split(flat, counts, top);
    }
    // discover_search_with_graph (search.rs:314-349): context stage for 10 entry points, then the discover search, in one call;
    // vectors = n_queries x (1 + 2 n_pairs) x dim (target, then the pairs)
    std::vector<std::vector<ScoredPointOffset>> search_discover(const float* vectors, uint32_t n_pairs, uint32_t n_queries, uint32_t top, uint32_t ef,
                                                                PointOffsetType entry_point, uint32_t entry_level, const uint64_t* deleted = nullptr,
                                                                SearchAlgorithm algorithm = SearchAlgorithm::Hnsw) const {
        std::vector<ScoredPointOffset> flat((size_t)n_queries * top);
        std::vector<uint32_t> counts(n_queries);
        check(qb_hnsw_search_discover_batch(h_, vectors, n_pairs, n_queries, top, ef, entry_point, entry_level, deleted, nullptr, flat.data(), counts.data(),
                                            nullptr, static_cast<qb_hnsw_algorithm>(algorithm)));
        return split(flat, counts, top);
    }
    // custom queries whose examples are multivectors, on a multivector graph (qb_hnsw_search_maxsim_custom_batch): example j of query q =
    // rows [example_offsets[q * E + j], example_offsets[q * E + j + 1]) of example_vectors; the rest as search_custom; deleted: over points
    std::vector<std::vector<ScoredPointOffset>> search_maxsim_custom(qb_query_kind kind, const float* example_vectors, const uint32_t* example_offsets,
                                                                     uint32_t n_a, uint32_t n_b, const float* coef, uint32_t n_queries, uint32_t top,
                                                                     uint32_t ef, PointOffsetType entry_point, uint32_t entry_level,
                                                                     const uint32_t* custom_entry_points = nullptr, const uint32_t* custom_counts = nullptr,
                                                                     uint32_t n_custom = 0, const uint64_t* deleted = nullptr,
                                                                     SearchAlgorithm algorithm = SearchAlgorithm::Hnsw) const {
        std::vector<ScoredPointOffset> flat((size_t)n_queries * top);
        std::vector<uint32_t> counts(n_queries);
        check(qb_hnsw_search_maxsim_custom_batch(h_, kind, example_vectors, example_offsets, n_a, n_b, coef, n_queries, top, ef, entry_point, entry_level,
                                                 custom_entry_points, custom_counts, n_custom, deleted, nullptr, flat.data(), counts.data(), nullptr,
                                                 static_cast<qb_hnsw_algorithm>(algorithm)));
        return split(flat, counts, top);
    }
    // discover with multivector examples, both stages in one call (qb_hnsw_search_maxsim_discover_batch); E = 1 + 2 n_pairs
    std::vector<std::vector<ScoredPointOffset>> search_maxsim_discover(const float* example_vectors, const uint32_t* example_offsets, uint32_t n_pairs,
                                                                       uint32_t n_queries, uint32_t top, uint32_t ef, PointOffsetType entry_point,
                                                                       uint32_t entry_level, const uint64_t* deleted = nullptr,
                                                                       SearchAlgorithm algorithm = SearchAlgorithm::Hnsw) const {
        std::vector<ScoredPointOffset> flat((size_t)n_queries * top);
        std::vector<uint32_t> counts(n_queries);
        check(qb_hnsw_search_maxsim_discover_batch(h_, example_vectors, example_offsets, n_pairs, n_queries, top, ef, entry_point, entry_level, deleted,
                                                   nullptr, flat.data(), counts.data(), nullptr, static_cast<qb_hnsw_algorithm>(algorithm)));
        return split(flat, counts, top);
    }

private:
    static std::vector<std::vector<ScoredPointOffset>> split(const std::vector<ScoredPointOffset>& flat, const std::vector<uint32_t>& counts, uint32_t top) {
        std::vector<std::vector<ScoredPointOffset>> out(counts.size());
        for (size_t q = 0; q < counts.size(); ++q) out[q].assign(flat.begin() + q * top, flat.begin() + q * top + counts[q]);
        return out;
    }
    explicit HnswGraph(qb_hnsw* h) : h_(h) {}
    qb_hnsw* h_ = nullptr;
};

// One shard (segment on one GPU) of a sharded search: SegmentsSearcher's blocking task per segment (segments_searcher.rs:255) calls
// search() with the same queries on every shard; the BatchResultAggregator step (search_result_aggregator.rs:50-117) happens on the
// devices and every call returns the merged top-k.  Wire the shards of one process with ShardedSegments::connect.
class SegmentShard {
public:
    SegmentShard(const VectorStorage& storage, int device, int rank, int world, uint32_t max_queries, uint32_t max_top) : st_(storage) {
        check(qb_comm_create(device, rank, world, max_queries, max_top, &c_));
    }
    ~SegmentShard() { qb_comm_destroy(c_); }
    SegmentShard(const SegmentShard&) = delete;
    static void connect(const std::vector<SegmentShard*>& shards) {
        std::vector<qb_comm*> cs;
        for (auto* s : shards) cs.push_back(s->c_);
        check(qb_comm_connect_local(cs.data(), (int32_t)cs.size()));
    }
    std::vector<std::vector<ScoredPointOffset>> search(const float* queries, uint32_t n_queries, uint32_t top) const {
        std::vector<ScoredPointOffset> flat((size_t)n_queries * top);
        std::vector<uint32_t> counts(n_queries);
        check(qb_multi_search_batch(c_, st_.raw(), queries, n_queries, top, nullptr, nullptr, flat.data(), counts.data(), nullptr));
        std::vector<std::vector<ScoredPointOffset>> out(n_queries);
        for (uint32_t q = 0; q < n_queries; ++q) out[q].assign(flat.begin() + (size_t)q * top, flat.begin() + (size_t)q * top + counts[q]);
        return out;
    }

private:
    const VectorStorage& st_;
    qb_comm* c_ = nullptr;
};

// A sparse vector: internal dims (the segment's IndicesTracker remapping) for SparseVectorIndex, user dims for SparseVectorStorage
struct SparseVector {
    std::vector<uint32_t> indices;
    std::vector<float> values;
};

// The inverted index of a sparse named vector and SearchContext over it (sparse/src/index/search_context.rs): search() is
// SearchContext::search, plain_search() is SearchContext::plain_search over already-filtered ids.  Ram may prune (InvertedIndexRam),
// Compressed never does (the compressed indexes with f32 weights).
class SparseVectorIndex {
public:
    enum class Kind : int { Ram = QB_SPARSE_RAM, Compressed = QB_SPARSE_COMPRESSED };
    SparseVectorIndex(const std::vector<SparseVector>& points, uint32_t n_dims, Kind kind = Kind::Ram, int device = 0) {
        std::vector<uint64_t> indptr(1, 0);
        std::vector<uint32_t> dims;
        std::vector<float> w;
        flatten(points, indptr, dims, w);
        check(qb_sparse_index_create(device, (qb_sparse_kind)kind, (uint32_t)points.size(), n_dims, indptr.data(), dims.data(), w.data(), &h_));
    }
    ~SparseVectorIndex() { qb_sparse_index_destroy(h_); }
    SparseVectorIndex(const SparseVectorIndex&) = delete;
    SparseVectorIndex& operator=(const SparseVectorIndex&) = delete;

    std::vector<std::vector<ScoredPointOffset>> search(const std::vector<SparseVector>& queries, uint32_t top, const uint64_t* deleted_bitmap = nullptr,
                                                       qb_hw_counters* counters = nullptr) const {
        std::vector<uint64_t> qp(1, 0);
        std::vector<uint32_t> qd;
        std::vector<float> qw;
        flatten(queries, qp, qd, qw);
        std::vector<ScoredPointOffset> flat(queries.size() * (size_t)top);
        std::vector<uint32_t> counts(queries.size());
        check(qb_sparse_search_batch(h_, qp.data(), qd.data(), qw.data(), (uint32_t)queries.size(), top, deleted_bitmap, nullptr, flat.data(), counts.data(),
                                     counters));
        return split(flat, counts, top);
    }
    std::vector<std::vector<ScoredPointOffset>> plain_search(const std::vector<SparseVector>& queries, const std::vector<std::vector<PointOffsetType>>& ids,
                                                             uint32_t top, qb_hw_counters* counters = nullptr) const {
        std::vector<uint64_t> qp(1, 0), ip(1, 0);
        std::vector<uint32_t> qd, flat_ids;
        std::vector<float> qw;
        flatten(queries, qp, qd, qw);
        for (const auto& l : ids) { flat_ids.insert(flat_ids.end(), l.begin(), l.end()); ip.push_back(flat_ids.size()); }
        if (ids.size() != queries.size()) throw OperationError(QB_ERR_INVALID, "plain_search: one id list per query");
        std::vector<ScoredPointOffset> flat(queries.size() * (size_t)top);
        std::vector<uint32_t> counts(queries.size());
        check(qb_sparse_search_plain_batch(h_, qp.data(), qd.data(), qw.data(), (uint32_t)queries.size(), ip.data(), flat_ids.data(), top, nullptr,
                                           flat.data(), counts.data(), counters));
        return split(flat, counts, top);
    }

private:
    friend class SparseVectorStorage;
    static void flatten(const std::vector<SparseVector>& v, std::vector<uint64_t>& ptr, std::vector<uint32_t>& dims, std::vector<float>& w) {
        for (const auto& x : v) {
            if (x.indices.size() != x.values.size()) throw OperationError(QB_ERR_INVALID, "sparse vector: indices and values differ in length");
            dims.insert(dims.end(), x.indices.begin(), x.indices.end());
            w.insert(w.end(), x.values.begin(), x.values.end());
            ptr.push_back(dims.size());
        }
    }
    static std::vector<std::vector<ScoredPointOffset>> split(const std::vector<ScoredPointOffset>& flat, const std::vector<uint32_t>& counts, uint32_t top) {
        std::vector<std::vector<ScoredPointOffset>> out(counts.size());
        for (size_t q = 0; q < counts.size(); ++q) out[q].assign(flat.begin() + q * top, flat.begin() + q * top + counts[q]);
        return out;
    }
    qb_sparse_index* h_ = nullptr;
};

// The sparse vector storage of a named vector, in user dims, and search_scored over it: the recommend / discover / context / feedback
// queries, which skip the inverted index (peek_top_iter with a SparseCustomQueryScorer).  One kind and shape per call: `examples` holds
// E = qb_custom_examples(kind, n_a, n_b) examples per query in the qb_scorer_create_custom order; `coef` [a, partial...] per query for
// feedback.  `id_list` (optional) is shared by the batch.
class SparseVectorStorage {
public:
    SparseVectorStorage(const std::vector<SparseVector>& points, bool on_disk = false, int device = 0) {
        std::vector<uint64_t> indptr(1, 0);
        std::vector<uint32_t> dims;
        std::vector<float> w;
        SparseVectorIndex::flatten(points, indptr, dims, w);
        check(qb_sparse_storage_create(device, (uint32_t)points.size(), indptr.data(), dims.data(), w.data(), on_disk ? 1 : 0, &h_));
    }
    ~SparseVectorStorage() { qb_sparse_storage_destroy(h_); }
    SparseVectorStorage(const SparseVectorStorage&) = delete;
    SparseVectorStorage& operator=(const SparseVectorStorage&) = delete;

    std::vector<std::vector<ScoredPointOffset>> search_custom(qb_query_kind kind, const std::vector<SparseVector>& examples, uint32_t n_a, uint32_t n_b,
                                                              const std::vector<float>* coef, uint32_t top, const uint64_t* deleted_bitmap = nullptr,
                                                              const std::vector<PointOffsetType>* id_list = nullptr, qb_hw_counters* counters = nullptr) const {
        std::vector<uint64_t> ep(1, 0);
        std::vector<uint32_t> ed;
        std::vector<float> ew;
        SparseVectorIndex::flatten(examples, ep, ed, ew);
        const uint32_t e = kind == QB_QUERY_RECO_BEST_SCORE || kind == QB_QUERY_RECO_SUM_SCORES ? n_a + n_b : kind == QB_QUERY_CONTEXT ? 2 * n_a : 1 + 2 * n_a;
        const size_t nq = e ? examples.size() / e : 0;
        std::vector<ScoredPointOffset> flat(nq * (size_t)top);
        std::vector<uint32_t> counts(nq);
        check(qb_sparse_search_custom_batch(h_, kind, n_a, n_b, ep.data(), ed.data(), ew.data(), coef ? coef->data() : nullptr, (uint32_t)nq, top, deleted_bitmap,
                                            id_list ? id_list->data() : nullptr, id_list ? id_list->size() : 0, nullptr, flat.data(), counts.data(), counters));
        return SparseVectorIndex::split(flat, counts, top);
    }
    std::vector<float> score_custom(qb_query_kind kind, const std::vector<SparseVector>& examples, uint32_t n_a, uint32_t n_b, const std::vector<float>* coef,
                                    const std::vector<PointOffsetType>& ids, qb_hw_counters* counters = nullptr) const {
        std::vector<uint64_t> ep(1, 0);
        std::vector<uint32_t> ed;
        std::vector<float> ew;
        SparseVectorIndex::flatten(examples, ep, ed, ew);
        std::vector<float> scores(ids.size());
        check(qb_sparse_score_custom(h_, kind, n_a, n_b, ep.data(), ed.data(), ew.data(), coef ? coef->data() : nullptr, ids.data(), ids.size(), scores.data(),
                                     counters));
        return scores;
    }
    // maximal marginal relevance over candidates whose sparse vectors are this storage's points: one query in user dims (any order),
    // (point id, score) candidates, pair scores score_vectors -> the selection, with the input scores
    std::vector<ScoredPointOffset> mmr(const SparseVector& query, const std::vector<ScoredPointOffset>& candidates, float lambda, uint32_t limit,
                                       qb_hw_counters* counters = nullptr) const {
        std::vector<uint64_t> qp(1, 0);
        std::vector<uint32_t> qd;
        std::vector<float> qw;
        SparseVectorIndex::flatten({query}, qp, qd, qw);
        std::vector<ScoredPointOffset> out(std::max<uint32_t>(limit, 1));
        const uint32_t n = (uint32_t)candidates.size();
        uint32_t count = 0;
        check(qb_mmr_sparse_batch(h_, qp.data(), qd.data(), qw.data(), 1, &lambda, candidates.data(), &n, n, limit, out.data(), &count, counters));
        out.resize(count);
        return out;
    }

private:
    qb_sparse_storage* h_ = nullptr;
};

}  // namespace qdrant_b200
