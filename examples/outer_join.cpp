// Outer joins on the data of the reference's examples/join.rs (String payloads replaced by indices into the tables
// below).  col1 has key 4 ("G","H"), which col2 lacks: the inner join drops it, r1.left_outer_join(r2) keeps it as
// (4, ((G,H), None)), and r2.right_outer_join(r1) as (4, (None, (G,H))).  Each join gives 7 rows; exit 0 only on the
// expected result.
#include <algorithm>
#include <cstdio>
#include <optional>
#include <string>

#include "vega_b200.hpp"

static const char *t1[] = {"(A,B)", "(C,D)", "(E,F)", "(G,H)"};
static const char *t2[] = {"A1", "A2", "B1", "B2", "C1", "C2"};

static std::string show(const std::optional<uint64_t> &x, const char *const *table)
{
    return x ? "Some(" + std::string(table[*x]) + ")" : "None";
}

int main()
{
    try {
        auto sc = vega::Context::create();
        std::vector<std::pair<int32_t, uint64_t>> col1 = {{1, 0}, {2, 1}, {3, 2}, {4, 3}};
        std::vector<std::pair<int32_t, uint64_t>> col2 = {{1, 0}, {1, 1}, {2, 2}, {2, 3}, {3, 4}, {3, 5}};
        auto r1 = sc->parallelize(col1, 4);
        auto r2 = sc->parallelize(col2, 4);

        auto left = r1.left_outer_join(r2, 4);
        std::sort(left.begin(), left.end());
        std::string s;
        for (auto &row : left)
            s += (s.empty() ? "" : ", ") + ("(" + std::to_string(row.first) + ", (" + t1[row.second.first] + ", " + show(row.second.second, t2) + "))");
        std::printf("left_outer_join: [%s]\n", s.c_str());
        const bool left_ok = left.size() == 7 && left.back().first == 4 && left.back().second.first == 3 && !left.back().second.second;

        auto right = r2.right_outer_join(r1, 4);
        std::sort(right.begin(), right.end());
        s.clear();
        for (auto &row : right)
            s += (s.empty() ? "" : ", ") + ("(" + std::to_string(row.first) + ", (" + show(row.second.first, t2) + ", " + t1[row.second.second] + "))");
        std::printf("right_outer_join: [%s]\n", s.c_str());
        const bool right_ok = right.size() == 7 && right.back().first == 4 && !right.back().second.first && right.back().second.second == 3;

        auto full = r1.full_outer_join(r2, 4);
        size_t none_w = 0, none_v = 0;
        for (auto &row : full) { none_v += !row.second.first; none_w += !row.second.second; }
        std::printf("full_outer_join: %zu rows, %zu without a right value, %zu without a left value\n", full.size(), none_w, none_v);
        const bool full_ok = full.size() == 7 && none_w == 1 && none_v == 0;

        return left_ok && right_ok && full_ok ? 0 : 1;
    } catch (const vega::Error &e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 2;
    }
}
