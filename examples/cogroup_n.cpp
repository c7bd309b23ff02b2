// cogroup and inner join of three parents (CoGroupedRdd with three dependencies), on small hand-written data:
//   a = (1,10) (2,20) (1,11) (5,50)   in 2 slices
//   b = (1,100) (3,300) (1,101)       in 1 slice
//   c = (1,1000) (2,2000) (3,3000)    in 2 slices
// The cogroup (3 partitions) gives every key once with one list per parent, in parent order; only key 1 is on all three
// parents, so the join is its 2 * 2 * 1 rows, the last parent varying fastest.  Exit 0 only on the expected result.
#include <algorithm>
#include <cstdio>
#include <string>

#include "vega_b200.hpp"

static std::string list(const std::vector<uint64_t> &xs)
{
    std::string s;
    for (uint64_t x : xs) s += (s.empty() ? "" : ", ") + std::to_string(x);
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

        auto cg = a.cogroup_n({b, c}, 3);
        std::sort(cg.begin(), cg.end());
        using Lists = std::vector<std::vector<uint64_t>>;
        const std::vector<std::pair<uint64_t, Lists>> want_cg = {
            {1, {{10, 11}, {100, 101}, {1000}}}, {2, {{20}, {}, {2000}}}, {3, {{}, {300}, {3000}}}, {5, {{50}, {}, {}}}};
        std::string s;
        for (const auto &[k, lists] : cg) {
            std::string ls;
            for (const auto &l : lists) ls += (ls.empty() ? "" : ", ") + list(l);
            s += (s.empty() ? "" : ", ") + ("(" + std::to_string(k) + ", [" + ls + "])");
        }
        std::printf("cogroup: [%s]\n", s.c_str());

        auto j = a.join_n({b, c}, 3);
        const std::vector<std::pair<uint64_t, std::vector<uint64_t>>> want_j = {
            {1, {10, 100, 1000}}, {1, {10, 101, 1000}}, {1, {11, 100, 1000}}, {1, {11, 101, 1000}}};
        s.clear();
        for (const auto &[k, vs] : j) s += (s.empty() ? "" : ", ") + ("(" + std::to_string(k) + ", " + list(vs) + ")");
        std::printf("join: [%s]\n", s.c_str());
        return cg == want_cg && j == want_j ? 0 : 1;
    } catch (const vega::Error &e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 2;
    }
}
