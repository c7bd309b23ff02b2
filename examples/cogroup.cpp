// cogroup on the data of the reference's tests/test_rdd.rs: the cogroup of (1,"A"), (2,"B"), (3,"C"), (4,"D") with
// itself (two slices, two partitions; the String payloads replaced by indices into the table below) gives every key
// once with ([X], [X]), and the cogroup behind intersection (col1 in 2 slices, col2 in 4, 3 partitions) keeps the keys
// with values on both sides: [3, 4, 5, 13]; the keys with an empty right list are the subtraction [0, 1, 2, 10, 12,
// 19].  Exit 0 only on the expected result.
#include <algorithm>
#include <cstdio>
#include <string>

#include "vega_b200.hpp"

static const char *names[] = {"A", "B", "C", "D"};

int main()
{
    try {
        auto sc = vega::Context::create();
        std::vector<std::pair<int32_t, uint64_t>> rows = {{1, 0}, {2, 1}, {3, 2}, {4, 3}};
        auto rdd0 = sc->parallelize(rows, 2);
        auto rdd1 = sc->parallelize(rows, 2);
        auto cg = rdd0.cogroup(rdd1, 2);
        std::sort(cg.begin(), cg.end());
        std::string s;
        bool cg_ok = cg.size() == 4;
        for (size_t i = 0; i < cg.size(); ++i) {
            const auto &[k, lists] = cg[i];
            const auto &[vs, ws] = lists;
            cg_ok = cg_ok && k == (int32_t)i + 1 && vs == std::vector<uint64_t>{i} && ws == vs;
            s += (s.empty() ? "" : ", ") + ("(" + std::to_string(k) + ", ([" + names[vs.at(0)] + "], [" + names[ws.at(0)] + "]))");
        }
        std::printf("cogroup: [%s]\n", s.c_str());

        std::vector<std::pair<int32_t, uint64_t>> col1, col2;
        for (int32_t x : {1, 2, 3, 4, 5, 10, 12, 13, 19, 0}) col1.emplace_back(x, 0);
        for (int32_t x : {3, 4, 5, 6, 7, 8, 11, 13}) col2.emplace_back(x, 0);
        auto both = sc->parallelize(col1, 2).cogroup(sc->parallelize(col2, 4), 3);
        std::vector<int32_t> inter, sub;
        for (const auto &[k, lists] : both) {
            if (!lists.first.empty() && !lists.second.empty()) inter.push_back(k);
            if (!lists.first.empty() && lists.second.empty()) sub.push_back(k);
        }
        std::sort(inter.begin(), inter.end());
        std::sort(sub.begin(), sub.end());
        s.clear();
        for (int32_t k : inter) s += (s.empty() ? "" : ", ") + std::to_string(k);
        std::printf("intersection: [%s]\n", s.c_str());
        s.clear();
        for (int32_t k : sub) s += (s.empty() ? "" : ", ") + std::to_string(k);
        std::printf("subtract: [%s]\n", s.c_str());
        const bool set_ok = inter == std::vector<int32_t>{3, 4, 5, 13} && sub == std::vector<int32_t>{0, 1, 2, 10, 12, 19} &&
                            both.size() == 14;
        return cg_ok && set_ok ? 0 : 1;
    } catch (const vega::Error &e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 2;
    }
}
