// The reference's examples/group_by.rs with its real String keys "x" and "y", plus a small word count
// (count_by_value over String words).  Expected output (the order of keys is unspecified; sorted here):
//   result: [("x", [1, 2, 3, 4, 5, 6, 7]), ("y", [1, 2, 3, 4, 5, 6, 7, 8])]
//   words: [("a", 2), ("be", 2), ("count", 1), ("is", 1), ("not", 1), ("of", 1), ("or", 1), ("question", 2), ("that", 1),
//           ("the", 1), ("to", 2), ("word", 1)]
#include <algorithm>
#include <cstdio>
#include <sstream>

#include "vega_b200.hpp"

int main()
{
    try {
        auto sc = vega::Context::create();
        std::vector<std::pair<std::string, int64_t>> vec;
        for (int i = 1; i <= 7; ++i) vec.emplace_back("x", i);
        for (int i = 1; i <= 8; ++i) vec.emplace_back("y", i);
        auto r = sc->make_rdd(vec, 4);
        auto res = r.group_by_key(4);
        std::sort(res.begin(), res.end());
        std::printf("result: [");
        for (size_t i = 0; i < res.size(); ++i) {
            std::printf("%s(\"%s\", [", i ? ", " : "", res[i].first.c_str());
            for (size_t j = 0; j < res[i].second.size(); ++j) std::printf("%s%lld", j ? ", " : "", (long long)res[i].second[j]);
            std::printf("])");
        }
        std::printf("]\n");
        bool ok = res.size() == 2 && res[0].first == "x" && res[1].first == "y" &&
                  res[0].second == std::vector<int64_t>{1, 2, 3, 4, 5, 6, 7} && res[1].second == std::vector<int64_t>{1, 2, 3, 4, 5, 6, 7, 8};

        // word count: count_by_value over the words of a line, and the same through reduce_by_key(sum) of (word, 1)
        std::istringstream text("to be or not to be that is the question a question of a word count");
        std::vector<std::string> words;
        for (std::string w; text >> w;) words.push_back(w);
        auto counts = sc->parallelize(words, 3).count_by_value();
        std::sort(counts.begin(), counts.end());
        std::vector<std::pair<std::string, uint64_t>> ones;
        for (auto &w : words) ones.emplace_back(w, 1);
        auto sums = sc->make_rdd(ones, 3).reduce_by_key(vega::Op::Sum, 2);
        std::sort(sums.begin(), sums.end());
        std::printf("words: [");
        for (size_t i = 0; i < counts.size(); ++i)
            std::printf("%s(\"%s\", %llu)", i ? ", " : "", counts[i].first.c_str(), (unsigned long long)counts[i].second);
        std::printf("]\n");
        uint64_t total = 0;
        for (auto &c : counts) total += c.second;
        ok = ok && total == words.size() && sums == counts && counts.size() == 12;
        for (auto &c : counts) ok = ok && c.second == (uint64_t)std::count(words.begin(), words.end(), c.first);
        return ok ? 0 : 1;
    } catch (const vega::Error &e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 2;
    }
}
