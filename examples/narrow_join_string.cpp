// Aggregate by word, then join by word, with no second shuffle: reduce_by_key(sum) of String keys kept on the device and
// joined under the same 3 partitions (CoGroupedRdd::new's OneToOneDependency, co_grouped_rdd.rs:103-112):
//   a = ("x",10) ("y",20) ("x",11) ("",50)    in 2 slices  ->  sums "x":21   "y":20   "":50
//   b = ("x",100) ("z",300) ("x",101) ("",5)  in 1 slice   ->  sums "x":201  "z":300  "":5
//   c = ("y",7) ("y",8)                       in 1 slice   ->  sums "y":15
// The join of the sums is ("", (50, 5)) and ("x", (21, 201)); the cogroup of all three gives every word once with the
// list [sum] from each result that has it; the outer join with only a required keeps a's words.  Exit 0 only on the
// expected rows.
#include <algorithm>
#include <cstdio>
#include <optional>
#include <string>

#include "vega_b200.hpp"

int main()
{
    try {
        auto sc = vega::Context::create();
        using Rows = std::vector<std::pair<std::string, uint64_t>>;
        auto a = sc->make_rdd(Rows{{"x", 10}, {"y", 20}, {"x", 11}, {"", 50}}, 2).reduce_by_key_rdd(vega::Op::Sum, 3);
        auto b = sc->make_rdd(Rows{{"x", 100}, {"z", 300}, {"x", 101}, {"", 5}}, 1).reduce_by_key_rdd(vega::Op::Sum, 3);
        auto c = sc->make_rdd(Rows{{"y", 7}, {"y", 8}}, 1).reduce_by_key_rdd(vega::Op::Sum, 3);

        auto j = a.join(b);
        std::sort(j.begin(), j.end());
        const std::vector<std::pair<std::string, std::pair<uint64_t, uint64_t>>> want_j = {{"", {50, 5}}, {"x", {21, 201}}};
        std::string s;
        for (const auto &[k, vw] : j)
            s += (s.empty() ? "" : ", ") + ("(\"" + k + "\", (" + std::to_string(vw.first) + ", " + std::to_string(vw.second) + "))");
        std::printf("join: [%s]\n", s.c_str());

        auto cg2 = a.cogroup(c);
        std::sort(cg2.begin(), cg2.end());
        using Pair = std::pair<std::vector<uint64_t>, std::vector<uint64_t>>;
        const std::vector<std::pair<std::string, Pair>> want_cg2 = {{"", {{50}, {}}}, {"x", {{21}, {}}}, {"y", {{20}, {15}}}};

        auto cg = a.cogroup_n({b, c});
        std::sort(cg.begin(), cg.end());
        using Lists = std::vector<std::vector<uint64_t>>;
        const std::vector<std::pair<std::string, Lists>> want_cg = {
            {"", {{50}, {5}, {}}}, {"x", {{21}, {201}, {}}}, {"y", {{20}, {}, {15}}}, {"z", {{}, {300}, {}}}};
        std::printf("cogroup: %zu keys\n", cg.size());

        auto oj = a.join_n_outer({b, c}, 1u);
        std::sort(oj.begin(), oj.end());
        using Row = std::vector<std::optional<uint64_t>>;
        const std::vector<std::pair<std::string, Row>> want_oj = {
            {"", {50, 5, std::nullopt}}, {"x", {21, 201, std::nullopt}}, {"y", {20, std::nullopt, 15}}};
        s.clear();
        for (const auto &[k, row] : oj) {
            std::string r;
            for (const auto &x : row) r += (r.empty() ? "" : ", ") + (x ? std::to_string(*x) : std::string("None"));
            s += (s.empty() ? "" : ", ") + ("(\"" + k + "\", [" + r + "])");
        }
        std::printf("left outer join: [%s]\n", s.c_str());

        auto sums = a.collect();
        std::sort(sums.begin(), sums.end());
        const std::vector<std::pair<std::string, uint64_t>> want_sums = {{"", 50}, {"x", 21}, {"y", 20}};
        return j == want_j && cg2 == want_cg2 && cg == want_cg && oj == want_oj && sums == want_sums ? 0 : 1;
    } catch (const vega::Error &e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 2;
    }
}
