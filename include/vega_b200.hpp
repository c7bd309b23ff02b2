// vega_b200.hpp — C++ host-side mirror of vega's operator API for the shuffle path, header-only,
// above the C ABI in vega_b200.h.  The reference is compiled Rust and its toolchain is absent from
// this image, so this is the compiled-language host layer: same names, argument meaning and error
// behaviour as the reference for the calls on the path —
//   Context::new / make_rdd / parallelize          src/context.rs:333-345,399-431
//   PairRdd::group_by_key / reduce_by_key / join   src/rdd/pair_rdd.rs:35-52,54-80,104-121
//   Rdd::count_by_value / distinct / collect       src/rdd/rdd.rs:450-459,502-522,420-434
//   Rdd::intersection / subtract                   src/rdd/rdd.rs:838-946
//   CoGroupedRdd::new over reduce results          src/rdd/co_grouped_rdd.rs:103-112 (OneToOneDependency; reduce_by_key_rdd,
//                                                  integer and String keys)
// Rows are Vec<(K,V)> with K in {u64,i64,i32,u32,std::string} and V in {u64,i64,f64}; std::string keys are placed
// like the reference's String keys and support group_by_key / reduce_by_key / count_by_key / count_by_value /
// distinct, and cogroup / join / outer joins of any number of parents.  reduce_by_key takes a named Op (the reference's serde_closure cannot cross into CUDA).  Errors throw vega::Error
// (the reference returns Result<_> / panics).
#pragma once
#include <cstdint>
#include <memory>
#include <optional>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "vega_b200.h"

namespace vega {

struct Error : std::runtime_error {
    int code;
    Error(int c, const std::string &m) : std::runtime_error("vega_b200 error " + std::to_string(c) + ": " + m), code(c) {}
};

inline void check(int rc)
{
    if (rc != VB_OK) throw Error(rc, vb_last_error());
}

enum class Op { Sum = VB_AGG_SUM, Min = VB_AGG_MIN, Max = VB_AGG_MAX };

namespace detail {
template <typename T> struct dtype;
template <> struct dtype<uint64_t> { static constexpr int code = VB_U64; static constexpr uint32_t width = 8; };
template <> struct dtype<int64_t> { static constexpr int code = VB_I64; static constexpr uint32_t width = 8; };
template <> struct dtype<uint32_t> { static constexpr int code = VB_U64; static constexpr uint32_t width = 4; };
template <> struct dtype<int32_t> { static constexpr int code = VB_I64; static constexpr uint32_t width = 4; };
template <> struct dtype<double> { static constexpr int code = VB_F64; static constexpr uint32_t width = 8; };

template <typename T> inline uint64_t to_bits(T v)
{
    if constexpr (std::is_same<T, double>::value) { uint64_t b; __builtin_memcpy(&b, &v, 8); return b; }
    else if constexpr (std::is_signed<T>::value) return (uint64_t)(int64_t)v;
    else return (uint64_t)v;
}
template <typename T> inline T from_bits(uint64_t b)
{
    if constexpr (std::is_same<T, double>::value) { double d; __builtin_memcpy(&d, &b, 8); return d; }
    else return (T)b;
}

struct ShufDeleter { void operator()(vb_shuf *s) const { vb_shuffle_free(s); } };
using ShufPtr = std::unique_ptr<vb_shuf, ShufDeleter>;
}  // namespace detail

class Context : public std::enable_shared_from_this<Context> {
public:
    // `Context::new()` (src/context.rs:333): here it opens CUDA device `device`.
    static std::shared_ptr<Context> create(int device = 0)
    {
        std::shared_ptr<Context> c(new Context());
        check(vb_ctx_create(device, &c->ctx_));
        return c;
    }
    ~Context() { if (ctx_) vb_ctx_destroy(ctx_); }
    vb_ctx *raw() const { return ctx_; }
    uint64_t new_shuffle_id() { return next_id_++; }

    template <typename K, typename V> class PairRddT;
    template <typename K, typename V> class ReducedRddT;
    template <typename K> class KeyRddT;

    template <typename K, typename V>
    PairRddT<K, V> make_rdd(const std::vector<std::pair<K, V>> &data, size_t num_slices);
    template <typename K, typename V>
    PairRddT<K, V> parallelize(const std::vector<std::pair<K, V>> &data, size_t num_slices) { return make_rdd(data, num_slices); }
    template <typename K> KeyRddT<K> parallelize(const std::vector<K> &data, size_t num_slices);

    // std::string keys (Rust String): group_by_key / reduce_by_key / count_by_key, count_by_value / distinct
    template <typename V> class StrPairRddT;
    template <typename V> class StrReducedRddT;
    class StrKeyRddT;
    template <typename V>
    StrPairRddT<V> make_rdd(const std::vector<std::pair<std::string, V>> &data, size_t num_slices);
    template <typename V>
    StrPairRddT<V> parallelize(const std::vector<std::pair<std::string, V>> &data, size_t num_slices) { return make_rdd(data, num_slices); }
    StrKeyRddT parallelize(const std::vector<std::string> &data, size_t num_slices);
    // byte-slice keys (Rust Vec<u8> / &[u8] / [u8; N]): the String-key RDDs with the keys placed as a Vec<u8> hashes
    // (vb_shuffle_set_str_key(VB_STRKEY_BYTES)); results carry each key's bytes in a std::string
    template <typename V>
    StrPairRddT<V> make_rdd(const std::vector<std::pair<std::vector<uint8_t>, V>> &data, size_t num_slices);
    template <typename V>
    StrPairRddT<V> parallelize(const std::vector<std::pair<std::vector<uint8_t>, V>> &data, size_t num_slices) { return make_rdd(data, num_slices); }
    StrKeyRddT parallelize(const std::vector<std::vector<uint8_t>> &data, size_t num_slices);

private:
    Context() = default;
    vb_ctx *ctx_ = nullptr;
    uint64_t next_id_ = 0;
};

namespace detail {
// Run one shuffle: slice like ParallelCollection::slice, one map task per slice, seal.  sorted_values: each key's list of
// a GROUP / COGROUP shuffle ascending in the value dtype's order (vb_shuffle_set_value_order).
template <typename K>
inline ShufPtr run_shuffle(Context &sc, const std::vector<uint64_t> &keys, const std::vector<uint64_t> *vals, size_t num_slices,
                           size_t num_splits, int vcode, int agg, bool sorted_values = false)
{
    if (num_slices < 1) throw Error(VB_ERR_INVALID, "Number of slices should be greater than or equal to 1");
    const uint64_t n = keys.size();
    std::vector<uint64_t> starts(std::min<uint64_t>(n, num_slices) + 2);
    const uint64_t n_map = vb_slice(n, num_slices, starts.data());
    vb_shuf *raw = nullptr;
    check(vb_shuffle_create(sc.raw(), sc.new_shuffle_id(), (uint32_t)n_map, (uint32_t)num_splits, dtype<K>::code, vcode, agg,
                            VB_PART_HASH_METRO64, &raw));
    ShufPtr s(raw);
    if (dtype<K>::width == 4) check(vb_shuffle_set_key_width(raw, 4));
    if (sorted_values) check(vb_shuffle_set_value_order(raw, VB_VALORDER_ASC));
    for (uint64_t m = 0; m < n_map; ++m) {
        const uint64_t lo = starts[m], cnt = starts[m + 1] - lo;
        check(vb_shuffle_map_soa(raw, (uint32_t)m, cnt ? keys.data() + lo : nullptr, (vals && cnt) ? vals->data() + lo : nullptr, cnt, VB_HOST));
    }
    check(vb_shuffle_seal(raw));
    return s;
}

// partitions [0, num_splits) of vb_cogroup_n over sealed sides  →  Vec<(K, Vec<Vec<V>>)>
template <typename K, typename V>
inline std::vector<std::pair<K, std::vector<std::vector<V>>>> read_cogroup_n(std::vector<vb_shuf *> sides, size_t num_splits)
{
    const uint32_t n = (uint32_t)sides.size();
    std::vector<std::pair<K, std::vector<std::vector<V>>>> out;
    for (uint32_t r = 0; r < num_splits; ++r) {
        uint64_t nk = 0;
        std::vector<uint64_t> nv(n);
        check(vb_cogroup_n_size(sides.data(), n, r, &nk, nv.data()));
        std::vector<uint64_t> k(nk);
        std::vector<std::vector<uint64_t>> offs(n, std::vector<uint64_t>(nk + 1)), vals(n);
        std::vector<uint64_t *> op(n);
        std::vector<void *> vp(n);
        for (uint32_t j = 0; j < n; ++j) { vals[j].resize(nv[j]); op[j] = offs[j].data(); vp[j] = vals[j].data(); }
        check(vb_cogroup_n(sides.data(), n, r, k.data(), op.data(), vp.data(), VB_HOST));
        for (uint64_t i = 0; i < nk; ++i) {
            std::vector<std::vector<V>> lists(n);
            for (uint32_t j = 0; j < n; ++j)
                for (uint64_t x = offs[j][i]; x < offs[j][i + 1]; ++x) lists[j].push_back(detail::from_bits<V>(vals[j][x]));
            out.emplace_back(detail::from_bits<K>(k[i]), std::move(lists));
        }
    }
    return out;
}

// partitions [0, num_splits) of vb_join_n_outer over sealed sides  →  (k, [v_0 or nullopt, ...]) per row
template <typename K, typename V>
inline std::vector<std::pair<K, std::vector<std::optional<V>>>> read_join_n_outer(std::vector<vb_shuf *> sides, size_t num_splits,
                                                                              uint32_t required)
{
    const uint32_t n = (uint32_t)sides.size();
    std::vector<std::pair<K, std::vector<std::optional<V>>>> out;
    for (uint32_t r = 0; r < num_splits; ++r) {
        uint64_t rows = 0;
        check(vb_join_n_outer_size(sides.data(), n, r, required, &rows));
        std::vector<uint64_t> k(rows);
        std::vector<std::vector<uint64_t>> vals(n, std::vector<uint64_t>(rows));
        std::vector<std::vector<uint8_t>> valid(n, std::vector<uint8_t>(rows));
        std::vector<void *> vp(n);
        std::vector<uint8_t *> ok(n);
        for (uint32_t j = 0; j < n; ++j) { vp[j] = vals[j].data(); ok[j] = valid[j].data(); }
        check(vb_join_n_outer(sides.data(), n, r, required, k.data(), vp.data(), ok.data(), VB_HOST));
        for (uint64_t i = 0; i < rows; ++i) {
            std::vector<std::optional<V>> row(n);
            for (uint32_t j = 0; j < n; ++j)
                if (valid[j][i]) row[j] = detail::from_bits<V>(vals[j][i]);
            out.emplace_back(detail::from_bits<K>(k[i]), std::move(row));
        }
    }
    return out;
}

// partitions [0, num_splits) of vb_semi_join_n over sealed sides  →  side 0's (k, v) rows of the kept keys
template <typename K, typename V>
inline std::vector<std::pair<K, V>> read_semi_join_n(std::vector<vb_shuf *> sides, size_t num_splits, uint32_t required,
                                                    uint32_t excluded)
{
    const uint32_t n = (uint32_t)sides.size();
    std::vector<std::pair<K, V>> out;
    for (uint32_t r = 0; r < num_splits; ++r) {
        uint64_t rows = 0;
        check(vb_semi_join_n_size(sides.data(), n, r, required, excluded, &rows));
        std::vector<uint64_t> k(rows), v(rows);
        check(vb_semi_join_n(sides.data(), n, r, required, excluded, k.data(), v.data(), VB_HOST));
        for (uint64_t i = 0; i < rows; ++i) out.emplace_back(detail::from_bits<K>(k[i]), detail::from_bits<V>(v[i]));
    }
    return out;
}
}  // namespace detail

template <typename K, typename V>
class Context::PairRddT {
public:
    PairRddT(std::shared_ptr<Context> sc, const std::vector<std::pair<K, V>> &data, size_t num_slices)
        : sc_(std::move(sc)), num_slices_(num_slices)
    {
        keys_.reserve(data.size());
        vals_.reserve(data.size());
        for (auto &kv : data) { keys_.push_back(detail::to_bits<K>(kv.first)); vals_.push_back(detail::to_bits<V>(kv.second)); }
    }
    size_t number_of_splits() const { return num_slices_; }

    // group_by_key(num_splits).collect()  →  Vec<(K, Vec<V>)>, values in input order, or ascending with sorted_values
    // (u64 unsigned, i64 signed, f64 as f64::total_cmp), sorted on the device
    std::vector<std::pair<K, std::vector<V>>> group_by_key(size_t num_splits, bool sorted_values = false) const
    {
        auto s = detail::run_shuffle<K>(*sc_, keys_, &vals_, num_slices_, num_splits, detail::dtype<V>::code, VB_AGG_GROUP, sorted_values);
        std::vector<std::pair<K, std::vector<V>>> out;
        for (uint32_t r = 0; r < num_splits; ++r) {
            uint64_t nk = 0, nv = 0;
            check(vb_shuffle_reduce_size(s.get(), r, &nk, &nv));
            std::vector<uint64_t> k(nk), o(nk + 1), v(nv);
            check(vb_shuffle_reduce(s.get(), r, k.data(), nullptr, o.data(), v.data(), VB_HOST));
            for (uint64_t i = 0; i < nk; ++i) {
                std::vector<V> vs;
                for (uint64_t j = o[i]; j < o[i + 1]; ++j) vs.push_back(detail::from_bits<V>(v[j]));
                out.emplace_back(detail::from_bits<K>(k[i]), std::move(vs));
            }
        }
        return out;
    }

    // reduce_by_key(op, num_splits).collect()  →  Vec<(K, V)>
    std::vector<std::pair<K, V>> reduce_by_key(Op op, size_t num_splits) const
    {
        auto s = detail::run_shuffle<K>(*sc_, keys_, &vals_, num_slices_, num_splits, detail::dtype<V>::code, (int)op);
        std::vector<std::pair<K, V>> out;
        for (uint32_t r = 0; r < num_splits; ++r) {
            uint64_t nk = 0, nv = 0;
            check(vb_shuffle_reduce_size(s.get(), r, &nk, &nv));
            std::vector<uint64_t> k(nk), c(nk);
            check(vb_shuffle_reduce(s.get(), r, k.data(), c.data(), nullptr, nullptr, VB_HOST));
            for (uint64_t i = 0; i < nk; ++i) out.emplace_back(detail::from_bits<K>(k[i]), detail::from_bits<V>(c[i]));
        }
        return out;
    }

    // reduce_by_key(op, num_splits) kept on the device: a ReducedRddT to collect, or to join / cogroup with other results
    // under the same num_splits without a second shuffle
    ReducedRddT<K, V> reduce_by_key_rdd(Op op, size_t num_splits) const
    {
        auto s = detail::run_shuffle<K>(*sc_, keys_, &vals_, num_slices_, num_splits, detail::dtype<V>::code, (int)op);
        return ReducedRddT<K, V>(std::shared_ptr<vb_shuf>(s.release(), detail::ShufDeleter()), num_splits);
    }

    // combine_by_key with named aggregates of the value column (VB_AGG_SUM / MIN / MAX / COUNT / MEAN), one shuffle:
    // per key one result per aggregate, as 64-bit patterns (COUNT: uint64_t, MEAN: double, others: V; read them with
    // detail::from_bits<T>)
    std::vector<std::pair<K, std::vector<uint64_t>>> combine_by_key(const std::vector<int32_t> &aggs, size_t num_splits) const
    {
        if (num_slices_ < 1) throw Error(VB_ERR_INVALID, "Number of slices should be greater than or equal to 1");
        const uint64_t n = keys_.size();
        std::vector<uint64_t> starts(std::min<uint64_t>(n, num_slices_) + 2);
        const uint64_t n_map = vb_slice(n, num_slices_, starts.data());
        std::vector<vb_agg_col> spec;
        for (int32_t a : aggs) spec.push_back(vb_agg_col{a, 0});
        const int32_t vcode = detail::dtype<V>::code;
        vb_shuf *raw = nullptr;
        check(vb_shuffle_create_multi(sc_->raw(), sc_->new_shuffle_id(), (uint32_t)n_map, (uint32_t)num_splits, detail::dtype<K>::code, 1,
                                      &vcode, (uint32_t)spec.size(), spec.data(), &raw));
        detail::ShufPtr s(raw);
        if (detail::dtype<K>::width == 4) check(vb_shuffle_set_key_width(raw, 4));
        for (uint64_t m = 0; m < n_map; ++m) {
            const uint64_t lo = starts[m], cnt = starts[m + 1] - lo;
            const void *col = cnt ? vals_.data() + lo : nullptr;
            check(vb_shuffle_map_cols(raw, (uint32_t)m, cnt ? keys_.data() + lo : nullptr, &col, cnt, VB_HOST));
        }
        check(vb_shuffle_seal(raw));
        std::vector<std::pair<K, std::vector<uint64_t>>> out;
        for (uint32_t r = 0; r < num_splits; ++r) {
            uint64_t nk = 0, nv = 0;
            check(vb_shuffle_reduce_size(raw, r, &nk, &nv));
            std::vector<uint64_t> k(nk);
            std::vector<std::vector<uint64_t>> cols(aggs.size(), std::vector<uint64_t>(nk));
            std::vector<void *> ptrs;
            for (auto &c : cols) ptrs.push_back(c.data());
            check(vb_shuffle_reduce_cols(raw, r, k.data(), ptrs.data(), VB_HOST));
            for (uint64_t i = 0; i < nk; ++i) {
                std::vector<uint64_t> row;
                for (auto &c : cols) row.push_back(c[i]);
                out.emplace_back(detail::from_bits<K>(k[i]), std::move(row));
            }
        }
        return out;
    }

    // self.join(other, num_splits).collect()  →  Vec<(K, (V, W))>, inner join.  sorted_values (here and in the cogroups
    // and joins below): every side's lists ascending, so a key's rows come in ascending (v, w) order.
    template <typename W>
    std::vector<std::pair<K, std::pair<V, W>>> join(const PairRddT<K, W> &other, size_t num_splits, bool sorted_values = false) const
    {
        auto a = detail::run_shuffle<K>(*sc_, keys_, &vals_, num_slices_, num_splits, detail::dtype<V>::code, VB_AGG_COGROUP, sorted_values);
        auto b = detail::run_shuffle<K>(*sc_, other.keys_, &other.vals_, other.num_slices_, num_splits, detail::dtype<W>::code, VB_AGG_COGROUP,
                                        sorted_values);
        std::vector<std::pair<K, std::pair<V, W>>> out;
        for (uint32_t r = 0; r < num_splits; ++r) {
            uint64_t n = 0;
            check(vb_join_size(a.get(), b.get(), r, &n));
            std::vector<uint64_t> k(n), v(n), w(n);
            check(vb_join(a.get(), b.get(), r, k.data(), v.data(), w.data(), VB_HOST));
            for (uint64_t i = 0; i < n; ++i)
                out.emplace_back(detail::from_bits<K>(k[i]), std::make_pair(detail::from_bits<V>(v[i]), detail::from_bits<W>(w[i])));
        }
        return out;
    }

    // self.cogroup(other, num_splits).collect()  →  Vec<(K, (Vec<V>, Vec<W>))> (src/rdd/pair_rdd.rs:123-155): every key
    // of either side once, with both value lists in cogroup order; a side that lacks the key has an empty list.
    template <typename W>
    std::vector<std::pair<K, std::pair<std::vector<V>, std::vector<W>>>> cogroup(const PairRddT<K, W> &other, size_t num_splits,
                                                                                 bool sorted_values = false) const
    {
        auto a = detail::run_shuffle<K>(*sc_, keys_, &vals_, num_slices_, num_splits, detail::dtype<V>::code, VB_AGG_COGROUP, sorted_values);
        auto b = detail::run_shuffle<K>(*sc_, other.keys_, &other.vals_, other.num_slices_, num_splits, detail::dtype<W>::code, VB_AGG_COGROUP,
                                        sorted_values);
        std::vector<std::pair<K, std::pair<std::vector<V>, std::vector<W>>>> out;
        for (uint32_t r = 0; r < num_splits; ++r) {
            uint64_t nk = 0, nv = 0, nw = 0;
            check(vb_cogroup_size(a.get(), b.get(), r, &nk, &nv, &nw));
            std::vector<uint64_t> k(nk), vo(nk + 1), v(nv), wo(nk + 1), w(nw);
            check(vb_cogroup(a.get(), b.get(), r, k.data(), vo.data(), v.data(), wo.data(), w.data(), VB_HOST));
            for (uint64_t i = 0; i < nk; ++i) {
                std::vector<V> vs;
                std::vector<W> ws;
                for (uint64_t j = vo[i]; j < vo[i + 1]; ++j) vs.push_back(detail::from_bits<V>(v[j]));
                for (uint64_t j = wo[i]; j < wo[i + 1]; ++j) ws.push_back(detail::from_bits<W>(w[j]));
                out.emplace_back(detail::from_bits<K>(k[i]), std::make_pair(std::move(vs), std::move(ws)));
            }
        }
        return out;
    }

    // Outer joins (Spark's leftOuterJoin / rightOuterJoin / fullOuterJoin; vega has none): a key missing on the other
    // side still gives rows, with std::nullopt on that side.  A key's rows are contiguous.
    template <typename W>
    std::vector<std::pair<K, std::pair<V, std::optional<W>>>> left_outer_join(const PairRddT<K, W> &other, size_t num_splits,
                                                       bool sorted_values = false) const
    {
        std::vector<std::pair<K, std::pair<V, std::optional<W>>>> out;
        outer_join_rows(other, num_splits, VB_JOIN_LEFT, sorted_values, [&](K k, std::optional<V> v, std::optional<W> w) { out.emplace_back(k, std::make_pair(*v, w)); });
        return out;
    }
    template <typename W>
    std::vector<std::pair<K, std::pair<std::optional<V>, W>>> right_outer_join(const PairRddT<K, W> &other, size_t num_splits,
                                                       bool sorted_values = false) const
    {
        std::vector<std::pair<K, std::pair<std::optional<V>, W>>> out;
        outer_join_rows(other, num_splits, VB_JOIN_RIGHT, sorted_values, [&](K k, std::optional<V> v, std::optional<W> w) { out.emplace_back(k, std::make_pair(v, *w)); });
        return out;
    }
    template <typename W>
    std::vector<std::pair<K, std::pair<std::optional<V>, std::optional<W>>>> full_outer_join(const PairRddT<K, W> &other, size_t num_splits,
                                                       bool sorted_values = false) const
    {
        std::vector<std::pair<K, std::pair<std::optional<V>, std::optional<W>>>> out;
        outer_join_rows(other, num_splits, VB_JOIN_FULL, sorted_values, [&](K k, std::optional<V> v, std::optional<W> w) { out.emplace_back(k, std::make_pair(v, w)); });
        return out;
    }

    // CoGroupedRdd::new([self, others...], HashPartitioner::new(num_splits)).collect()  →  Vec<(K, Vec<Vec<V>>)>
    // (src/rdd/co_grouped_rdd.rs:75-135, 206-249): every key of any parent once, with one value list per parent in
    // parent order (this one first); a parent that lacks the key has an empty list.
    std::vector<std::pair<K, std::vector<std::vector<V>>>> cogroup_n(const std::vector<PairRddT> &others, size_t num_splits,
                                                                     bool sorted_values = false) const
    {
        auto shs = cogroup_shuffles(others, num_splits, sorted_values);
        std::vector<vb_shuf *> sides;
        for (auto &s : shs) sides.push_back(s.get());
        return detail::read_cogroup_n<K, V>(sides, num_splits);
    }

    // inner join of [self, others...]  →  (k, [v_0, ..., v_{n-1}]) per row: for a key on every parent,
    // for v0 in vs_0 { for v1 in vs_1 { ... } }
    std::vector<std::pair<K, std::vector<V>>> join_n(const std::vector<PairRddT> &others, size_t num_splits, bool sorted_values = false) const
    {
        auto shs = cogroup_shuffles(others, num_splits, sorted_values);
        std::vector<vb_shuf *> sides;
        for (auto &s : shs) sides.push_back(s.get());
        const uint32_t n = (uint32_t)sides.size();
        std::vector<std::pair<K, std::vector<V>>> out;
        for (uint32_t r = 0; r < num_splits; ++r) {
            uint64_t rows = 0;
            check(vb_join_n_size(sides.data(), n, r, &rows));
            std::vector<uint64_t> k(rows);
            std::vector<std::vector<uint64_t>> vals(n, std::vector<uint64_t>(rows));
            std::vector<void *> vp(n);
            for (uint32_t j = 0; j < n; ++j) vp[j] = vals[j].data();
            check(vb_join_n(sides.data(), n, r, k.data(), vp.data(), VB_HOST));
            for (uint64_t i = 0; i < rows; ++i) {
                std::vector<V> row(n);
                for (uint32_t j = 0; j < n; ++j) row[j] = detail::from_bits<V>(vals[j][i]);
                out.emplace_back(detail::from_bits<K>(k[i]), std::move(row));
            }
        }
        return out;
    }

    // outer join of [self, others...] (vega has none): bit j of `required` marks parent j (this one is 0) required.  A
    // key on every required parent gives, for v0 in L0 { for v1 in L1 { ... } }, (k, [v_0, ..., v_{n-1}]) where L_j is
    // parent j's list, or [std::nullopt] for an optional parent that lacks the key.  A key's rows are contiguous.
    std::vector<std::pair<K, std::vector<std::optional<V>>>> join_n_outer(const std::vector<PairRddT> &others, size_t num_splits,
                                                                          uint32_t required, bool sorted_values = false) const
    {
        auto shs = cogroup_shuffles(others, num_splits, sorted_values);
        std::vector<vb_shuf *> sides;
        for (auto &s : shs) sides.push_back(s.get());
        return detail::read_join_n_outer<K, V>(sides, num_splits, required);
    }

    // semi / anti join of this parent by [others...] (vega has none): bit j of `required` / `excluded` marks parent j
    // (1 .. n-1; this one is 0) as a parent that must / must not have the key.  A kept key gives its (k, v) rows of this
    // parent, contiguous and in list order.  The other parents' values are never read and their lazy rows never grouped.
    std::vector<std::pair<K, V>> semi_join_n(const std::vector<PairRddT> &others, size_t num_splits, uint32_t required,
                                             uint32_t excluded, bool sorted_values = false) const
    {
        auto shs = cogroup_shuffles(others, num_splits, sorted_values);
        std::vector<vb_shuf *> sides;
        for (auto &s : shs) sides.push_back(s.get());
        return detail::read_semi_join_n<K, V>(sides, num_splits, required, excluded);
    }
    // Spark's subtractByKey: this parent's rows whose key `other` lacks
    std::vector<std::pair<K, V>> subtract_by_key(const PairRddT &other, size_t num_splits, bool sorted_values = false) const
    {
        return semi_join_n({other}, num_splits, 0, 0b10, sorted_values);
    }
    // left semi join: this parent's rows whose key `other` has, each once
    std::vector<std::pair<K, V>> semi_join(const PairRddT &other, size_t num_splits, bool sorted_values = false) const
    {
        return semi_join_n({other}, num_splits, 0b10, 0, sorted_values);
    }

    std::shared_ptr<Context> sc_;
    size_t num_slices_;
    std::vector<uint64_t> keys_, vals_;

private:
    // one COGROUP shuffle per parent: this one, then others in order
    std::vector<detail::ShufPtr> cogroup_shuffles(const std::vector<PairRddT> &others, size_t num_splits, bool sorted_values) const
    {
        std::vector<detail::ShufPtr> shs;
        shs.push_back(detail::run_shuffle<K>(*sc_, keys_, &vals_, num_slices_, num_splits, detail::dtype<V>::code, VB_AGG_COGROUP, sorted_values));
        for (auto &o : others)
            shs.push_back(detail::run_shuffle<K>(*sc_, o.keys_, &o.vals_, o.num_slices_, num_splits, detail::dtype<V>::code, VB_AGG_COGROUP,
                                                 sorted_values));
        return shs;
    }

    // every row of vb_join_outer, partition by partition, as emit(k, v or nullopt, w or nullopt)
    template <typename W, typename Emit>
    void outer_join_rows(const PairRddT<K, W> &other, size_t num_splits, int32_t kind, bool sorted_values, Emit emit) const
    {
        auto a = detail::run_shuffle<K>(*sc_, keys_, &vals_, num_slices_, num_splits, detail::dtype<V>::code, VB_AGG_COGROUP, sorted_values);
        auto b = detail::run_shuffle<K>(*sc_, other.keys_, &other.vals_, other.num_slices_, num_splits, detail::dtype<W>::code, VB_AGG_COGROUP,
                                        sorted_values);
        for (uint32_t r = 0; r < num_splits; ++r) {
            uint64_t n = 0;
            check(vb_join_outer_size(a.get(), b.get(), r, kind, &n));
            std::vector<uint64_t> k(n), v(n), w(n);
            std::vector<uint8_t> vv(n), wv(n);
            check(vb_join_outer(a.get(), b.get(), r, kind, k.data(), v.data(), w.data(), vv.data(), wv.data(), VB_HOST));
            for (uint64_t i = 0; i < n; ++i)
                emit(detail::from_bits<K>(k[i]), vv[i] ? std::optional<V>(detail::from_bits<V>(v[i])) : std::nullopt,
                     wv[i] ? std::optional<W>(detail::from_bits<W>(w[i])) : std::nullopt);
        }
    }
};

// A sealed reduce_by_key result on the device (PairRddT::reduce_by_key_rdd).  Partition r holds the keys with
// hash % num_splits == r, each once, so as a join / cogroup parent under the same num_splits it is read through a view
// (vb_shuffle_create_narrow: CoGroupedRdd::new's OneToOneDependency, co_grouped_rdd.rs:103-112) and not shuffled again;
// each key's list is [its result].  Parents of a join / cogroup must have the same num_splits (vega::Error otherwise).
template <typename K, typename V>
class Context::ReducedRddT {
public:
    ReducedRddT(std::shared_ptr<vb_shuf> s, size_t num_splits) : s_(std::move(s)), num_splits_(num_splits) {}
    size_t number_of_splits() const { return num_splits_; }

    // collect()  →  Vec<(K, V)>
    std::vector<std::pair<K, V>> collect() const
    {
        std::vector<std::pair<K, V>> out;
        for (uint32_t r = 0; r < num_splits_; ++r) {
            uint64_t nk = 0, nv = 0;
            check(vb_shuffle_reduce_size(s_.get(), r, &nk, &nv));
            std::vector<uint64_t> k(nk), c(nk);
            check(vb_shuffle_reduce(s_.get(), r, k.data(), c.data(), nullptr, nullptr, VB_HOST));
            for (uint64_t i = 0; i < nk; ++i) out.emplace_back(detail::from_bits<K>(k[i]), detail::from_bits<V>(c[i]));
        }
        return out;
    }

    // self.join(other).collect()  →  Vec<(K, (V, W))>: the keys both results have, with both results
    template <typename W>
    std::vector<std::pair<K, std::pair<V, W>>> join(const ReducedRddT<K, W> &other) const
    {
        auto a = view(*this), b = view(other);
        std::vector<std::pair<K, std::pair<V, W>>> out;
        for (uint32_t r = 0; r < num_splits_; ++r) {
            uint64_t n = 0;
            check(vb_join_size(a.get(), b.get(), r, &n));
            std::vector<uint64_t> k(n), v(n), w(n);
            check(vb_join(a.get(), b.get(), r, k.data(), v.data(), w.data(), VB_HOST));
            for (uint64_t i = 0; i < n; ++i)
                out.emplace_back(detail::from_bits<K>(k[i]), std::make_pair(detail::from_bits<V>(v[i]), detail::from_bits<W>(w[i])));
        }
        return out;
    }

    // CoGroupedRdd::new([self, others...]).collect()  →  Vec<(K, Vec<Vec<V>>)>: every key of any result once, with the
    // list [result] from each result that has it and [] from the others
    std::vector<std::pair<K, std::vector<std::vector<V>>>> cogroup_n(const std::vector<ReducedRddT> &others) const
    {
        auto views = views_of(others);
        return detail::read_cogroup_n<K, V>(raw(views), num_splits_);
    }

    // outer join of [self, others...] with PairRddT::join_n_outer's `required` bitmask and row order
    std::vector<std::pair<K, std::vector<std::optional<V>>>> join_n_outer(const std::vector<ReducedRddT> &others, uint32_t required) const
    {
        auto views = views_of(others);
        return detail::read_join_n_outer<K, V>(raw(views), num_splits_, required);
    }

    std::shared_ptr<vb_shuf> s_;
    size_t num_splits_;

private:
    template <typename W>
    detail::ShufPtr view(const ReducedRddT<K, W> &p) const
    {
        if (p.num_splits_ != num_splits_) throw Error(VB_ERR_INVALID, "join / cogroup parents of reduce results need the same num_splits");
        vb_shuf *v = nullptr;
        check(vb_shuffle_create_narrow(p.s_.get(), 0, &v));
        return detail::ShufPtr(v);
    }
    std::vector<detail::ShufPtr> views_of(const std::vector<ReducedRddT> &others) const
    {
        std::vector<detail::ShufPtr> vs;
        vs.push_back(view(*this));
        for (auto &o : others) vs.push_back(view(o));
        return vs;
    }
    static std::vector<vb_shuf *> raw(const std::vector<detail::ShufPtr> &vs)
    {
        std::vector<vb_shuf *> r;
        for (auto &v : vs) r.push_back(v.get());
        return r;
    }
};

template <typename K>
class Context::KeyRddT {
public:
    KeyRddT(std::shared_ptr<Context> sc, const std::vector<K> &data, size_t num_slices) : sc_(std::move(sc)), num_slices_(num_slices)
    {
        for (auto &k : data) keys_.push_back(detail::to_bits<K>(k));
    }
    // count_by_value().collect() → Vec<(K, u64)>   (src/rdd/rdd.rs:450-459)
    std::vector<std::pair<K, uint64_t>> count_by_value() const
    {
        std::vector<uint64_t> starts(std::min<uint64_t>(keys_.size(), num_slices_) + 2);
        const size_t n_splits = vb_slice(keys_.size(), num_slices_, starts.data());
        auto s = detail::run_shuffle<K>(*sc_, keys_, nullptr, num_slices_, n_splits, VB_U64, VB_AGG_COUNT);
        std::vector<std::pair<K, uint64_t>> out;
        for (uint32_t r = 0; r < n_splits; ++r) {
            uint64_t nk = 0, nv = 0;
            check(vb_shuffle_reduce_size(s.get(), r, &nk, &nv));
            std::vector<uint64_t> k(nk), c(nk);
            check(vb_shuffle_reduce(s.get(), r, k.data(), c.data(), nullptr, nullptr, VB_HOST));
            for (uint64_t i = 0; i < nk; ++i) out.emplace_back(detail::from_bits<K>(k[i]), c[i]);
        }
        return out;
    }
    // intersection(other[, num_splits]).collect() / subtract(other).collect()   (src/rdd/rdd.rs:838-946): the reference
    // cogroups (x, None) of both sides and reads the two Vec lengths; here ONE tagged SUM shuffle — side A rows carry 1,
    // side B rows 2^32 — so a key's sum says on which sides it occurred.  Each key once, like the reference.
    std::vector<K> intersection(const KeyRddT<K> &other, size_t num_splits = 0) const { return set_op(other, num_splits, true); }
    std::vector<K> subtract(const KeyRddT<K> &other, size_t num_splits = 0) const { return set_op(other, num_splits, false); }

    // distinct().collect()   (src/rdd/rdd.rs:502-522)
    std::vector<K> distinct() const
    {
        std::vector<K> out;
        for (auto &kv : count_by_value()) out.push_back(kv.first);
        return out;
    }

private:
    std::vector<K> set_op(const KeyRddT<K> &other, size_t num_splits, bool both) const
    {
        std::vector<uint64_t> sa(std::min<uint64_t>(keys_.size(), num_slices_) + 2), sb(std::min<uint64_t>(other.keys_.size(), other.num_slices_) + 2);
        const uint64_t na = vb_slice(keys_.size(), num_slices_, sa.data()), nb = vb_slice(other.keys_.size(), other.num_slices_, sb.data());
        if (num_splits == 0) num_splits = (size_t)na;                       // self.number_of_splits()
        vb_shuf *raw = nullptr;
        check(vb_shuffle_create(sc_->raw(), sc_->new_shuffle_id(), (uint32_t)(na + nb), (uint32_t)num_splits, detail::dtype<K>::code, VB_U64,
                                VB_AGG_SUM, VB_PART_HASH_METRO64, &raw));
        detail::ShufPtr s(raw);
        if (detail::dtype<K>::width == 4) check(vb_shuffle_set_key_width(raw, 4));
        const std::vector<uint64_t> ta(keys_.size(), 1ull), tb(other.keys_.size(), 1ull << 32);
        for (uint64_t m = 0; m < na; ++m)
            check(vb_shuffle_map_soa(raw, (uint32_t)m, keys_.data() + sa[m], ta.data() + sa[m], sa[m + 1] - sa[m], VB_HOST));
        for (uint64_t m = 0; m < nb; ++m)
            check(vb_shuffle_map_soa(raw, (uint32_t)(na + m), other.keys_.data() + sb[m], tb.data() + sb[m], sb[m + 1] - sb[m], VB_HOST));
        check(vb_shuffle_seal(raw));
        std::vector<K> out;
        for (uint32_t r = 0; r < num_splits; ++r) {
            uint64_t nk = 0, nv = 0;
            check(vb_shuffle_reduce_size(raw, r, &nk, &nv));
            std::vector<uint64_t> k(nk), c(nk);
            check(vb_shuffle_reduce(raw, r, k.data(), c.data(), nullptr, nullptr, VB_HOST));
            for (uint64_t i = 0; i < nk; ++i) {
                const bool in_a = (c[i] & 0xFFFFFFFFull) != 0, in_b = (c[i] >> 32) != 0;
                if (both ? (in_a && in_b) : (in_a && !in_b)) out.push_back(detail::from_bits<K>(k[i]));
            }
        }
        return out;
    }

    std::shared_ptr<Context> sc_;
    size_t num_slices_;
    std::vector<uint64_t> keys_;
};

namespace detail {
// A string key column, Arrow-style: key i is bytes[offs[i] .. offs[i + 1]).
struct StrCol {
    std::vector<uint64_t> offs{0};
    std::string bytes;
    int32_t kind = VB_STRKEY_STR;         // how the shuffles of this column place its keys (vb_shuffle_set_str_key)
    void push(const std::string &k) { bytes += k; offs.push_back(bytes.size()); }
    void push(const std::vector<uint8_t> &k) { bytes.append(k.begin(), k.end()); offs.push_back(bytes.size()); }
    uint64_t size() const { return offs.size() - 1; }
};

inline ShufPtr run_str_shuffle(Context &sc, const StrCol &keys, const std::vector<uint64_t> *vals, size_t num_slices, size_t num_splits,
                               int vcode, int agg, bool sorted_values = false)
{
    if (num_slices < 1) throw Error(VB_ERR_INVALID, "Number of slices should be greater than or equal to 1");
    const uint64_t n = keys.size();
    std::vector<uint64_t> starts(std::min<uint64_t>(n, num_slices) + 2);
    const uint64_t n_map = vb_slice(n, num_slices, starts.data());
    vb_shuf *raw = nullptr;
    check(vb_shuffle_create_str(sc.raw(), sc.new_shuffle_id(), (uint32_t)n_map, (uint32_t)num_splits, vcode, agg, &raw));
    ShufPtr s(raw);
    if (keys.kind != VB_STRKEY_STR) check(vb_shuffle_set_str_key(raw, keys.kind));
    if (sorted_values) check(vb_shuffle_set_value_order(raw, VB_VALORDER_ASC));
    for (uint64_t m = 0; m < n_map; ++m) {
        const uint64_t lo = starts[m], cnt = starts[m + 1] - lo;
        check(vb_shuffle_map_str(raw, (uint32_t)m, keys.offs.data() + lo, keys.bytes.data(), keys.bytes.size(),
                                 (vals && cnt) ? vals->data() + lo : nullptr, cnt, VB_HOST));
    }
    check(vb_shuffle_seal(raw));
    return s;
}

// partition r of a sealed string shuffle: its keys, and the combined values (reduce ops) or the CSR (GROUP)
inline std::vector<std::string> read_str_part(vb_shuf *s, uint32_t r, std::vector<uint64_t> *comb, std::vector<uint64_t> *offs,
                                              std::vector<uint64_t> *vals)
{
    uint64_t nk = 0, nb = 0, nv = 0;
    check(vb_shuffle_reduce_str_size(s, r, &nk, &nb, &nv));
    std::vector<uint64_t> ko(nk + 1);
    std::string kb(nb, '\0');
    if (comb) comb->resize(nk);
    if (offs) offs->resize(nk + 1);
    if (vals) vals->resize(nv);
    check(vb_shuffle_reduce_str(s, r, ko.data(), kb.data(), comb ? comb->data() : nullptr, offs ? offs->data() : nullptr,
                                vals ? vals->data() : nullptr, VB_HOST));
    std::vector<std::string> keys;
    for (uint64_t i = 0; i < nk; ++i) keys.emplace_back(kb, ko[i], ko[i + 1] - ko[i]);
    return keys;
}

// CoGroupedRdd::compute over String keys (vb_cogroup_n_str) of sealed string GROUP sides, partition by partition: every
// key of any side once, with one value list per side
template <typename V>
inline std::vector<std::pair<std::string, std::vector<std::vector<V>>>> read_str_cogroup_n(const std::vector<vb_shuf *> &sides,
                                                                                           size_t num_splits)
{
    const uint32_t n = (uint32_t)sides.size();
    std::vector<std::pair<std::string, std::vector<std::vector<V>>>> out;
    for (uint32_t r = 0; r < num_splits; ++r) {
        uint64_t nk = 0, nb = 0;
        std::vector<uint64_t> nv(n);
        check(vb_cogroup_n_str_size(sides.data(), n, r, &nk, &nb, nv.data()));
        std::vector<uint64_t> ko(nk + 1);
        std::string kb(nb, '\0');
        std::vector<std::vector<uint64_t>> offs(n, std::vector<uint64_t>(nk + 1)), vals(n);
        std::vector<uint64_t *> op(n);
        std::vector<void *> vp(n);
        for (uint32_t j = 0; j < n; ++j) { vals[j].resize(nv[j]); op[j] = offs[j].data(); vp[j] = vals[j].data(); }
        check(vb_cogroup_n_str(sides.data(), n, r, ko.data(), kb.data(), op.data(), vp.data(), VB_HOST));
        for (uint64_t i = 0; i < nk; ++i) {
            std::vector<std::vector<V>> lists(n);
            for (uint32_t j = 0; j < n; ++j)
                for (uint64_t x = offs[j][i]; x < offs[j][i + 1]; ++x) lists[j].push_back(from_bits<V>(vals[j][x]));
            out.emplace_back(std::string(kb, ko[i], ko[i + 1] - ko[i]), std::move(lists));
        }
    }
    return out;
}

// the outer join (vb_join_n_str) of sealed string GROUP sides with `required`, partition by partition:
// (k, [v_0, ..., v_{n-1}]) per row, std::nullopt where an optional side lacks the key
template <typename V>
inline std::vector<std::pair<std::string, std::vector<std::optional<V>>>> read_str_join_n_outer(const std::vector<vb_shuf *> &sides,
                                                                                                size_t num_splits, uint32_t required)
{
    const uint32_t n = (uint32_t)sides.size();
    std::vector<std::pair<std::string, std::vector<std::optional<V>>>> out;
    for (uint32_t r = 0; r < num_splits; ++r) {
        uint64_t rows = 0, nk = 0, nb = 0;
        check(vb_join_n_str_size(sides.data(), n, r, required, &rows, &nk, &nb));
        std::vector<uint64_t> ko(nk + 1), ro(nk + 1);
        std::string kb(nb, '\0');
        std::vector<std::vector<uint64_t>> vals(n, std::vector<uint64_t>(rows));
        std::vector<std::vector<uint8_t>> valid(n, std::vector<uint8_t>(rows));
        std::vector<void *> vp(n);
        std::vector<uint8_t *> ok(n);
        for (uint32_t j = 0; j < n; ++j) { vp[j] = vals[j].data(); ok[j] = valid[j].data(); }
        check(vb_join_n_str(sides.data(), n, r, required, ko.data(), kb.data(), ro.data(), vp.data(), ok.data(), VB_HOST));
        for (uint64_t i = 0; i < nk; ++i) {
            const std::string k(kb, ko[i], ko[i + 1] - ko[i]);
            for (uint64_t x = ro[i]; x < ro[i + 1]; ++x) {
                std::vector<std::optional<V>> row(n);
                for (uint32_t j = 0; j < n; ++j)
                    if (valid[j][x]) row[j] = from_bits<V>(vals[j][x]);
                out.emplace_back(k, std::move(row));
            }
        }
    }
    return out;
}

// vb_semi_join_n_str over sealed string GROUP sides, partition by partition: side 0's (k, v) rows of the kept keys
template <typename V>
inline std::vector<std::pair<std::string, V>> read_str_semi_join_n(const std::vector<vb_shuf *> &sides, size_t num_splits,
                                                                   uint32_t required, uint32_t excluded)
{
    const uint32_t n = (uint32_t)sides.size();
    std::vector<std::pair<std::string, V>> out;
    for (uint32_t r = 0; r < num_splits; ++r) {
        uint64_t rows = 0, nk = 0, nb = 0;
        check(vb_semi_join_n_str_size(sides.data(), n, r, required, excluded, &rows, &nk, &nb));
        std::vector<uint64_t> ko(nk + 1), ro(nk + 1), v(rows);
        std::string kb(nb, '\0');
        check(vb_semi_join_n_str(sides.data(), n, r, required, excluded, ko.data(), kb.data(), ro.data(), v.data(), VB_HOST));
        for (uint64_t i = 0; i < nk; ++i) {
            const std::string k(kb, ko[i], ko[i + 1] - ko[i]);
            for (uint64_t x = ro[i]; x < ro[i + 1]; ++x) out.emplace_back(k, from_bits<V>(v[x]));
        }
    }
    return out;
}
}  // namespace detail

template <typename V>
class Context::StrPairRddT {
public:
    StrPairRddT(std::shared_ptr<Context> sc, const std::vector<std::pair<std::string, V>> &data, size_t num_slices)
        : sc_(std::move(sc)), num_slices_(num_slices)
    {
        for (auto &kv : data) { keys_.push(kv.first); vals_.push_back(detail::to_bits<V>(kv.second)); }
    }
    StrPairRddT(std::shared_ptr<Context> sc, const std::vector<std::pair<std::vector<uint8_t>, V>> &data, size_t num_slices)
        : sc_(std::move(sc)), num_slices_(num_slices)
    {
        keys_.kind = VB_STRKEY_BYTES;
        for (auto &kv : data) { keys_.push(kv.first); vals_.push_back(detail::to_bits<V>(kv.second)); }
    }
    size_t number_of_splits() const { return num_slices_; }

    // group_by_key(num_splits).collect()  →  Vec<(String, Vec<V>)>, values in input order, or ascending with sorted_values
    std::vector<std::pair<std::string, std::vector<V>>> group_by_key(size_t num_splits, bool sorted_values = false) const
    {
        auto s = detail::run_str_shuffle(*sc_, keys_, &vals_, num_slices_, num_splits, detail::dtype<V>::code, VB_AGG_GROUP, sorted_values);
        std::vector<std::pair<std::string, std::vector<V>>> out;
        for (uint32_t r = 0; r < num_splits; ++r) {
            std::vector<uint64_t> o, v;
            auto k = detail::read_str_part(s.get(), r, nullptr, &o, &v);
            for (size_t i = 0; i < k.size(); ++i) {
                std::vector<V> vs;
                for (uint64_t j = o[i]; j < o[i + 1]; ++j) vs.push_back(detail::from_bits<V>(v[j]));
                out.emplace_back(std::move(k[i]), std::move(vs));
            }
        }
        return out;
    }

    // reduce_by_key(op, num_splits).collect()  →  Vec<(String, V)>
    std::vector<std::pair<std::string, V>> reduce_by_key(Op op, size_t num_splits) const
    {
        auto s = detail::run_str_shuffle(*sc_, keys_, &vals_, num_slices_, num_splits, detail::dtype<V>::code, (int)op);
        std::vector<std::pair<std::string, V>> out;
        for (uint32_t r = 0; r < num_splits; ++r) {
            std::vector<uint64_t> c;
            auto k = detail::read_str_part(s.get(), r, &c, nullptr, nullptr);
            for (size_t i = 0; i < k.size(); ++i) out.emplace_back(std::move(k[i]), detail::from_bits<V>(c[i]));
        }
        return out;
    }

    // reduce_by_key(op, num_splits) kept on the device: a StrReducedRddT to collect, or to join / cogroup with other
    // results under the same num_splits without a second shuffle
    StrReducedRddT<V> reduce_by_key_rdd(Op op, size_t num_splits) const
    {
        auto s = detail::run_str_shuffle(*sc_, keys_, &vals_, num_slices_, num_splits, detail::dtype<V>::code, (int)op);
        return StrReducedRddT<V>(std::shared_ptr<vb_shuf>(s.release(), detail::ShufDeleter()), num_splits);
    }

    // count_by_key(num_splits).collect()  →  Vec<(String, u64)>
    std::vector<std::pair<std::string, uint64_t>> count_by_key(size_t num_splits) const
    {
        auto s = detail::run_str_shuffle(*sc_, keys_, nullptr, num_slices_, num_splits, VB_U64, VB_AGG_COUNT);
        std::vector<std::pair<std::string, uint64_t>> out;
        for (uint32_t r = 0; r < num_splits; ++r) {
            std::vector<uint64_t> c;
            auto k = detail::read_str_part(s.get(), r, &c, nullptr, nullptr);
            for (size_t i = 0; i < k.size(); ++i) out.emplace_back(std::move(k[i]), c[i]);
        }
        return out;
    }

    // combine_by_key with named aggregates of the value column (VB_AGG_SUM / MIN / MAX / COUNT / MEAN) over String keys,
    // one shuffle (vb_shuffle_create_str_multi): per key one result per aggregate, as 64-bit patterns (COUNT: uint64_t,
    // MEAN: double, others: V; read them with detail::from_bits<T>)
    std::vector<std::pair<std::string, std::vector<uint64_t>>> combine_by_key(const std::vector<int32_t> &aggs, size_t num_splits) const
    {
        if (num_slices_ < 1) throw Error(VB_ERR_INVALID, "Number of slices should be greater than or equal to 1");
        const uint64_t n = keys_.size();
        std::vector<uint64_t> starts(std::min<uint64_t>(n, num_slices_) + 2);
        const uint64_t n_map = vb_slice(n, num_slices_, starts.data());
        std::vector<vb_agg_col> spec;
        for (int32_t a : aggs) spec.push_back(vb_agg_col{a, 0});
        const int32_t vcode = detail::dtype<V>::code;
        vb_shuf *raw = nullptr;
        check(vb_shuffle_create_str_multi(sc_->raw(), sc_->new_shuffle_id(), (uint32_t)n_map, (uint32_t)num_splits, 1, &vcode,
                                          (uint32_t)spec.size(), spec.data(), &raw));
        detail::ShufPtr s(raw);
        if (keys_.kind != VB_STRKEY_STR) check(vb_shuffle_set_str_key(raw, keys_.kind));
        for (uint64_t m = 0; m < n_map; ++m) {
            const uint64_t lo = starts[m], cnt = starts[m + 1] - lo;
            const void *col = cnt ? vals_.data() + lo : nullptr;
            check(vb_shuffle_map_str_cols(raw, (uint32_t)m, keys_.offs.data() + lo, keys_.bytes.data(), keys_.bytes.size(), &col, cnt,
                                          VB_HOST));
        }
        check(vb_shuffle_seal(raw));
        std::vector<std::pair<std::string, std::vector<uint64_t>>> out;
        for (uint32_t r = 0; r < num_splits; ++r) {
            uint64_t nk = 0, nb = 0;
            check(vb_shuffle_reduce_str_size(raw, r, &nk, &nb, nullptr));
            std::vector<uint64_t> ko(nk + 1);
            std::string kb(nb, '\0');
            std::vector<std::vector<uint64_t>> cols(aggs.size(), std::vector<uint64_t>(nk));
            std::vector<void *> ptrs;
            for (auto &c : cols) ptrs.push_back(c.data());
            check(vb_shuffle_reduce_str_cols(raw, r, ko.data(), kb.data(), ptrs.data(), VB_HOST));
            for (uint64_t i = 0; i < nk; ++i) {
                std::vector<uint64_t> row;
                for (auto &c : cols) row.push_back(c[i]);
                out.emplace_back(std::string(kb, ko[i], ko[i + 1] - ko[i]), std::move(row));
            }
        }
        return out;
    }

    // CoGroupedRdd::new([self, others...], HashPartitioner::new(num_splits)).collect() over String keys
    // (vb_cogroup_n_str): every key of any parent once, with one value list per parent (this one first)
    std::vector<std::pair<std::string, std::vector<std::vector<V>>>> cogroup_n(const std::vector<StrPairRddT> &others,
                                                                               size_t num_splits, bool sorted_values = false) const
    {
        auto shs = group_shuffles(others, num_splits, sorted_values);
        return detail::read_str_cogroup_n<V>(raw(shs), num_splits);
    }

    // outer join of [self, others...] (vb_join_n_str): bit j of `required` marks parent j (this one is 0) required;
    // an optional parent that lacks the key gives std::nullopt.  (k, [v_0, ..., v_{n-1}]) per row, a key's rows
    // contiguous, for v0 in L0 { for v1 in L1 { ... } }
    std::vector<std::pair<std::string, std::vector<std::optional<V>>>> join_n_outer(const std::vector<StrPairRddT> &others,
                                                                                    size_t num_splits, uint32_t required,
                                                                                    bool sorted_values = false) const
    {
        auto shs = group_shuffles(others, num_splits, sorted_values);
        return detail::read_str_join_n_outer<V>(raw(shs), num_splits, required);
    }

    // PairRddT::semi_join_n over String keys (vb_semi_join_n_str), keys matched by their bytes
    std::vector<std::pair<std::string, V>> semi_join_n(const std::vector<StrPairRddT> &others, size_t num_splits, uint32_t required,
                                                       uint32_t excluded, bool sorted_values = false) const
    {
        auto shs = group_shuffles(others, num_splits, sorted_values);
        return detail::read_str_semi_join_n<V>(raw(shs), num_splits, required, excluded);
    }
    std::vector<std::pair<std::string, V>> subtract_by_key(const StrPairRddT &other, size_t num_splits, bool sorted_values = false) const
    {
        return semi_join_n({other}, num_splits, 0, 0b10, sorted_values);
    }
    std::vector<std::pair<std::string, V>> semi_join(const StrPairRddT &other, size_t num_splits, bool sorted_values = false) const
    {
        return semi_join_n({other}, num_splits, 0b10, 0, sorted_values);
    }

    // inner join of [self, others...]  →  (k, [v_0, ..., v_{n-1}]) per row
    std::vector<std::pair<std::string, std::vector<V>>> join_n(const std::vector<StrPairRddT> &others, size_t num_splits,
                                                               bool sorted_values = false) const
    {
        std::vector<std::pair<std::string, std::vector<V>>> out;
        for (auto &kv : join_n_outer(others, num_splits, (uint32_t)((1ull << (others.size() + 1)) - 1), sorted_values)) {
            std::vector<V> row;
            for (auto &v : kv.second) row.push_back(*v);
            out.emplace_back(std::move(kv.first), std::move(row));
        }
        return out;
    }

    // PairRdd::join (src/rdd/pair_rdd.rs:104-121)  →  Vec<(String, (V, V))>
    std::vector<std::pair<std::string, std::pair<V, V>>> join(const StrPairRddT &other, size_t num_splits, bool sorted_values = false) const
    {
        std::vector<std::pair<std::string, std::pair<V, V>>> out;
        for (auto &kv : join_n({other}, num_splits, sorted_values)) out.emplace_back(std::move(kv.first), std::make_pair(kv.second[0], kv.second[1]));
        return out;
    }

    // PairRdd::cogroup (src/rdd/pair_rdd.rs:123-155)  →  Vec<(String, (Vec<V>, Vec<V>))>
    std::vector<std::pair<std::string, std::pair<std::vector<V>, std::vector<V>>>> cogroup(const StrPairRddT &other, size_t num_splits,
                                                                                           bool sorted_values = false) const
    {
        std::vector<std::pair<std::string, std::pair<std::vector<V>, std::vector<V>>>> out;
        for (auto &kv : cogroup_n({other}, num_splits, sorted_values))
            out.emplace_back(std::move(kv.first), std::make_pair(std::move(kv.second[0]), std::move(kv.second[1])));
        return out;
    }

private:
    // this parent and the others, each shuffled into a string GROUP shuffle over num_splits
    std::vector<detail::ShufPtr> group_shuffles(const std::vector<StrPairRddT> &others, size_t num_splits, bool sorted_values) const
    {
        std::vector<detail::ShufPtr> shs;
        shs.push_back(detail::run_str_shuffle(*sc_, keys_, &vals_, num_slices_, num_splits, detail::dtype<V>::code, VB_AGG_GROUP, sorted_values));
        for (auto &o : others)
            shs.push_back(detail::run_str_shuffle(*o.sc_, o.keys_, &o.vals_, o.num_slices_, num_splits, detail::dtype<V>::code, VB_AGG_GROUP,
                                                  sorted_values));
        return shs;
    }
    static std::vector<vb_shuf *> raw(const std::vector<detail::ShufPtr> &shs)
    {
        std::vector<vb_shuf *> out;
        for (auto &s : shs) out.push_back(s.get());
        return out;
    }

    std::shared_ptr<Context> sc_;
    size_t num_slices_;
    detail::StrCol keys_;
    std::vector<uint64_t> vals_;
};

// A sealed String reduce_by_key result on the device (StrPairRddT::reduce_by_key_rdd).  Partition r holds the keys with
// vb_hash_str(key) % num_splits == r, each once, so as a join / cogroup parent under the same num_splits it is read
// through a view (vb_shuffle_create_narrow_str: CoGroupedRdd::new's OneToOneDependency, co_grouped_rdd.rs:103-112) and
// not shuffled again; each key's list is [its result].  Parents of a join / cogroup must have the same num_splits
// (vega::Error otherwise).
template <typename V>
class Context::StrReducedRddT {
public:
    StrReducedRddT(std::shared_ptr<vb_shuf> s, size_t num_splits) : s_(std::move(s)), num_splits_(num_splits) {}
    size_t number_of_splits() const { return num_splits_; }

    // collect()  →  Vec<(String, V)>
    std::vector<std::pair<std::string, V>> collect() const
    {
        std::vector<std::pair<std::string, V>> out;
        for (uint32_t r = 0; r < num_splits_; ++r) {
            std::vector<uint64_t> c;
            auto k = detail::read_str_part(s_.get(), r, &c, nullptr, nullptr);
            for (size_t i = 0; i < k.size(); ++i) out.emplace_back(std::move(k[i]), detail::from_bits<V>(c[i]));
        }
        return out;
    }

    // self.join(other).collect()  →  Vec<(String, (V, W))>: the keys both results have, with both results
    template <typename W>
    std::vector<std::pair<std::string, std::pair<V, W>>> join(const StrReducedRddT<W> &other) const
    {
        auto a = view(*this), b = view(other);
        std::vector<std::pair<std::string, std::pair<V, W>>> out;
        for (auto &kv : detail::read_str_join_n_outer<uint64_t>({a.get(), b.get()}, num_splits_, 0b11))
            out.emplace_back(std::move(kv.first), std::make_pair(detail::from_bits<V>(*kv.second[0]), detail::from_bits<W>(*kv.second[1])));
        return out;
    }

    // self.cogroup(other).collect()  →  Vec<(String, (Vec<V>, Vec<W>))>: every key of either result once, with the list
    // [result] from a result that has it and [] from the other
    template <typename W>
    std::vector<std::pair<std::string, std::pair<std::vector<V>, std::vector<W>>>> cogroup(const StrReducedRddT<W> &other) const
    {
        auto a = view(*this), b = view(other);
        std::vector<std::pair<std::string, std::pair<std::vector<V>, std::vector<W>>>> out;
        for (auto &kv : detail::read_str_cogroup_n<uint64_t>({a.get(), b.get()}, num_splits_)) {
            std::vector<V> vs;
            std::vector<W> ws;
            for (uint64_t x : kv.second[0]) vs.push_back(detail::from_bits<V>(x));
            for (uint64_t x : kv.second[1]) ws.push_back(detail::from_bits<W>(x));
            out.emplace_back(std::move(kv.first), std::make_pair(std::move(vs), std::move(ws)));
        }
        return out;
    }

    // CoGroupedRdd::new([self, others...]).collect()  →  Vec<(String, Vec<Vec<V>>)>: every key of any result once, with
    // the list [result] from each result that has it and [] from the others
    std::vector<std::pair<std::string, std::vector<std::vector<V>>>> cogroup_n(const std::vector<StrReducedRddT> &others) const
    {
        auto views = views_of(others);
        return detail::read_str_cogroup_n<V>(raw(views), num_splits_);
    }

    // outer join of [self, others...] with StrPairRddT::join_n_outer's `required` bitmask and row order
    std::vector<std::pair<std::string, std::vector<std::optional<V>>>> join_n_outer(const std::vector<StrReducedRddT> &others,
                                                                                    uint32_t required) const
    {
        auto views = views_of(others);
        return detail::read_str_join_n_outer<V>(raw(views), num_splits_, required);
    }

    std::shared_ptr<vb_shuf> s_;
    size_t num_splits_;

private:
    template <typename W>
    detail::ShufPtr view(const StrReducedRddT<W> &p) const
    {
        if (p.num_splits_ != num_splits_) throw Error(VB_ERR_INVALID, "join / cogroup parents of reduce results need the same num_splits");
        vb_shuf *v = nullptr;
        check(vb_shuffle_create_narrow_str(p.s_.get(), 0, &v));
        return detail::ShufPtr(v);
    }
    std::vector<detail::ShufPtr> views_of(const std::vector<StrReducedRddT> &others) const
    {
        std::vector<detail::ShufPtr> vs;
        vs.push_back(view(*this));
        for (auto &o : others) vs.push_back(view(o));
        return vs;
    }
    static std::vector<vb_shuf *> raw(const std::vector<detail::ShufPtr> &vs)
    {
        std::vector<vb_shuf *> r;
        for (auto &v : vs) r.push_back(v.get());
        return r;
    }
};

class Context::StrKeyRddT {
public:
    StrKeyRddT(std::shared_ptr<Context> sc, const std::vector<std::string> &data, size_t num_slices) : sc_(std::move(sc)), num_slices_(num_slices)
    {
        for (auto &k : data) keys_.push(k);
    }
    StrKeyRddT(std::shared_ptr<Context> sc, const std::vector<std::vector<uint8_t>> &data, size_t num_slices)
        : sc_(std::move(sc)), num_slices_(num_slices)
    {
        keys_.kind = VB_STRKEY_BYTES;
        for (auto &k : data) keys_.push(k);
    }
    // count_by_value().collect() → Vec<(String, u64)>   (src/rdd/rdd.rs:450-459)
    std::vector<std::pair<std::string, uint64_t>> count_by_value() const
    {
        std::vector<uint64_t> starts(std::min<uint64_t>(keys_.size(), num_slices_) + 2);
        const size_t n_splits = vb_slice(keys_.size(), num_slices_, starts.data());
        auto s = detail::run_str_shuffle(*sc_, keys_, nullptr, num_slices_, n_splits, VB_U64, VB_AGG_COUNT);
        std::vector<std::pair<std::string, uint64_t>> out;
        for (uint32_t r = 0; r < n_splits; ++r) {
            std::vector<uint64_t> c;
            auto k = detail::read_str_part(s.get(), r, &c, nullptr, nullptr);
            for (size_t i = 0; i < k.size(); ++i) out.emplace_back(std::move(k[i]), c[i]);
        }
        return out;
    }
    // distinct().collect()   (src/rdd/rdd.rs:502-522)
    std::vector<std::string> distinct() const
    {
        std::vector<std::string> out;
        for (auto &kv : count_by_value()) out.push_back(kv.first);
        return out;
    }

private:
    std::shared_ptr<Context> sc_;
    size_t num_slices_;
    detail::StrCol keys_;
};

template <typename V>
Context::StrPairRddT<V> Context::make_rdd(const std::vector<std::pair<std::string, V>> &data, size_t num_slices)
{
    return StrPairRddT<V>(shared_from_this(), data, num_slices);
}
inline Context::StrKeyRddT Context::parallelize(const std::vector<std::string> &data, size_t num_slices)
{
    return StrKeyRddT(shared_from_this(), data, num_slices);
}
template <typename V>
Context::StrPairRddT<V> Context::make_rdd(const std::vector<std::pair<std::vector<uint8_t>, V>> &data, size_t num_slices)
{
    return StrPairRddT<V>(shared_from_this(), data, num_slices);
}
inline Context::StrKeyRddT Context::parallelize(const std::vector<std::vector<uint8_t>> &data, size_t num_slices)
{
    return StrKeyRddT(shared_from_this(), data, num_slices);
}

template <typename K, typename V>
Context::PairRddT<K, V> Context::make_rdd(const std::vector<std::pair<K, V>> &data, size_t num_slices)
{
    return PairRddT<K, V>(shared_from_this(), data, num_slices);
}
template <typename K>
Context::KeyRddT<K> Context::parallelize(const std::vector<K> &data, size_t num_slices)
{
    return KeyRddT<K>(shared_from_this(), data, num_slices);
}

}  // namespace vega
