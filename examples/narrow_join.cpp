// Aggregate, then join, with no second shuffle: reduce_by_key(sum) of two small hand-written inputs kept on the device
// and joined under the same 3 partitions (CoGroupedRdd::new's OneToOneDependency, co_grouped_rdd.rs:103-112):
//   a = (1,10) (2,20) (1,11) (5,50)    in 2 slices  ->  sums 1:21   2:20   5:50
//   b = (1,100) (3,300) (1,101) (5,5)  in 1 slice   ->  sums 1:201  3:300  5:5
//   c = (2,7) (2,8)                    in 1 slice   ->  sums 2:15
// The join of the sums is (1, (21, 201)) and (5, (50, 5)); the cogroup of all three gives every key once with the list
// [sum] from each result that has it; the outer join with only a required keeps a's keys.  Exit 0 only on the expected rows.
#include <algorithm>
#include <cstdio>
#include <optional>
#include <string>

#include "vega_b200.hpp"

int main()
{
    try {
        auto sc = vega::Context::create();
        using Rows = std::vector<std::pair<uint64_t, uint64_t>>;
        auto a = sc->parallelize(Rows{{1, 10}, {2, 20}, {1, 11}, {5, 50}}, 2).reduce_by_key_rdd(vega::Op::Sum, 3);
        auto b = sc->parallelize(Rows{{1, 100}, {3, 300}, {1, 101}, {5, 5}}, 1).reduce_by_key_rdd(vega::Op::Sum, 3);
        auto c = sc->parallelize(Rows{{2, 7}, {2, 8}}, 1).reduce_by_key_rdd(vega::Op::Sum, 3);

        auto j = a.join(b);
        std::sort(j.begin(), j.end());
        const std::vector<std::pair<uint64_t, std::pair<uint64_t, uint64_t>>> want_j = {{1, {21, 201}}, {5, {50, 5}}};
        std::string s;
        for (const auto &[k, vw] : j)
            s += (s.empty() ? "" : ", ") + ("(" + std::to_string(k) + ", (" + std::to_string(vw.first) + ", " + std::to_string(vw.second) + "))");
        std::printf("join: [%s]\n", s.c_str());

        auto cg = a.cogroup_n({b, c});
        std::sort(cg.begin(), cg.end());
        using Lists = std::vector<std::vector<uint64_t>>;
        const std::vector<std::pair<uint64_t, Lists>> want_cg = {
            {1, {{21}, {201}, {}}}, {2, {{20}, {}, {15}}}, {3, {{}, {300}, {}}}, {5, {{50}, {5}, {}}}};
        std::printf("cogroup: %zu keys\n", cg.size());

        auto oj = a.join_n_outer({b, c}, 1u);
        std::sort(oj.begin(), oj.end());
        using Row = std::vector<std::optional<uint64_t>>;
        const std::vector<std::pair<uint64_t, Row>> want_oj = {
            {1, {21, 201, std::nullopt}}, {2, {20, std::nullopt, 15}}, {5, {50, 5, std::nullopt}}};
        s.clear();
        for (const auto &[k, row] : oj) {
            std::string r;
            for (const auto &x : row) r += (r.empty() ? "" : ", ") + (x ? std::to_string(*x) : std::string("None"));
            s += (s.empty() ? "" : ", ") + ("(" + std::to_string(k) + ", [" + r + "])");
        }
        std::printf("left outer join: [%s]\n", s.c_str());
        return j == want_j && cg == want_cg && oj == want_oj ? 0 : 1;
    } catch (const vega::Error &e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 2;
    }
}
