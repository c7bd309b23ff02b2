// The reference's tests/test_pair_rdd.rs group_by data ("x" 1..7, "y" 1..8) cogrouped and joined with a second
// String-key RDD, plus one left outer join.  Expected output (the order of keys is unspecified; sorted here):
//   cogroup: [("x", ([1, 2, 3, 4, 5, 6, 7], [10, 11])), ("y", ([1, 2, 3, 4, 5, 6, 7, 8], [30])), ("z", ([], [20]))]
//   join ok: 22 rows
//   left outer join ok: 23 rows
#include <algorithm>
#include <cstdio>

#include "vega_b200.hpp"

int main()
{
    try {
        auto sc = vega::Context::create();
        std::vector<std::pair<std::string, int64_t>> vec;
        for (int i = 1; i <= 7; ++i) vec.emplace_back("x", i);
        for (int i = 1; i <= 8; ++i) vec.emplace_back("y", i);
        auto a = sc->make_rdd(vec, 4);
        auto b = sc->make_rdd(std::vector<std::pair<std::string, int64_t>>{{"x", 10}, {"z", 20}, {"y", 30}, {"x", 11}}, 2);

        auto cg = a.cogroup(b, 4);
        std::sort(cg.begin(), cg.end());
        auto list = [](const std::vector<int64_t> &v) {
            std::string s = "[";
            for (size_t i = 0; i < v.size(); ++i) s += (i ? ", " : "") + std::to_string(v[i]);
            return s + "]";
        };
        std::printf("cogroup: [");
        for (size_t i = 0; i < cg.size(); ++i)
            std::printf("%s(\"%s\", (%s, %s))", i ? ", " : "", cg[i].first.c_str(), list(cg[i].second.first).c_str(),
                        list(cg[i].second.second).c_str());
        std::printf("]\n");
        bool ok = cg.size() == 3 && cg[2].first == "z" && cg[2].second.first.empty();

        // inner join: x gives 7 * 2 rows, y 8 * 1, z none
        auto j = a.join(b, 4);
        std::sort(j.begin(), j.end());
        std::vector<std::pair<std::string, std::pair<int64_t, int64_t>>> want;
        for (int v = 1; v <= 7; ++v) { want.push_back({"x", {v, 10}}); want.push_back({"x", {v, 11}}); }
        for (int v = 1; v <= 8; ++v) want.push_back({"y", {v, 30}});
        std::sort(want.begin(), want.end());
        const bool join_ok = j == want;
        if (join_ok) std::printf("join ok: %zu rows\n", j.size());

        // left outer join of b with a: every key of b, "z" with None on a's side
        auto lo = b.join_n_outer({a}, 4, 0b01);
        size_t nz = 0, none = 0;
        for (auto &row : lo) {
            nz += row.first == "z";
            none += !row.second[1].has_value();
        }
        const bool left_ok = lo.size() == 23 && nz == 1 && none == 1;
        if (left_ok) std::printf("left outer join ok: %zu rows\n", lo.size());
        return ok && join_ok && left_ok ? 0 : 1;
    } catch (const vega::Error &e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 2;
    }
}
