// outer joins of three parents (CoGroupedRdd with three dependencies, expanded with None for a missing optional parent),
// on the data of examples/cogroup_n.cpp:
//   a = (1,10) (2,20) (1,11) (5,50)   in 2 slices
//   b = (1,100) (3,300) (1,101)       in 1 slice
//   c = (1,1000) (2,2000) (3,3000)    in 2 slices
// required = 0b001 is `a LEFT JOIN b LEFT JOIN c`: every key of a, with None where b or c lacks it.  required = 0 is the
// full outer join: key 3 (on b and c only) is kept too.  A key's rows come in nested order, the last parent varying
// fastest; the order of keys is unspecified, so the rows are sorted by key, stably.  Exit 0 only on the expected result.
#include <algorithm>
#include <cstdio>
#include <string>

#include "vega_b200.hpp"

using Row = std::pair<uint64_t, std::vector<std::optional<uint64_t>>>;

static std::string show(const std::vector<Row> &rows)
{
    std::string s;
    for (const auto &[k, vs] : rows) {
        std::string l;
        for (const auto &v : vs) l += (l.empty() ? "" : ", ") + (v ? std::to_string(*v) : std::string("None"));
        s += (s.empty() ? "" : ", ") + ("(" + std::to_string(k) + ", [" + l + "])");
    }
    return "[" + s + "]";
}

int main()
{
    try {
        auto sc = vega::Context::create();
        using Rows = std::vector<std::pair<uint64_t, uint64_t>>;
        auto a = sc->parallelize(Rows{{1, 10}, {2, 20}, {1, 11}, {5, 50}}, 2);
        auto b = sc->parallelize(Rows{{1, 100}, {3, 300}, {1, 101}}, 1);
        auto c = sc->parallelize(Rows{{1, 1000}, {2, 2000}, {3, 3000}}, 2);
        const auto none = std::nullopt;
        const std::vector<Row> key1 = {{1, {10, 100, 1000}}, {1, {10, 101, 1000}}, {1, {11, 100, 1000}}, {1, {11, 101, 1000}}};
        std::vector<Row> want_left = key1, want_full = key1;
        want_left.insert(want_left.end(), {{2, {20, none, 2000}}, {5, {50, none, none}}});
        want_full.insert(want_full.end(), {{2, {20, none, 2000}}, {3, {none, 300, 3000}}, {5, {50, none, none}}});
        const auto by_key = [](const Row &x, const Row &y) { return x.first < y.first; };

        auto left = a.join_n_outer({b, c}, 3, 0b001);
        std::stable_sort(left.begin(), left.end(), by_key);
        std::printf("left: %s\n", show(left).c_str());
        auto full = a.join_n_outer({b, c}, 3, 0);
        std::stable_sort(full.begin(), full.end(), by_key);
        std::printf("full: %s\n", show(full).c_str());
        return left == want_left && full == want_full ? 0 : 1;
    } catch (const vega::Error &e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 2;
    }
}
