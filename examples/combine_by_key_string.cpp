// combine_by_key over String keys: the per-word count, sum, min, max and mean of a value column from ONE shuffle that
// encodes every word once (vb_shuffle_create_str_multi).  Expected output (sorted by key):
//   result: [("", n=2, sum=-3, min=-5, max=2, mean=-1.5), ("x", n=7, sum=28, min=1, max=7, mean=4),
//            ("y", n=8, sum=36, min=1, max=8, mean=4.5), ("日本", n=1, sum=9, min=9, max=9, mean=9)]
//   ok
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
        vec.emplace_back("", 2);
        vec.emplace_back("", -5);
        vec.emplace_back("日本", 9);
        auto r = sc->make_rdd(vec, 4);
        auto res = r.combine_by_key({VB_AGG_COUNT, VB_AGG_SUM, VB_AGG_MIN, VB_AGG_MAX, VB_AGG_MEAN}, 3);
        std::sort(res.begin(), res.end());
        struct Want { const char *k; uint64_t n; int64_t sum, lo, hi; double mean; };
        const Want want[] = {{"", 2, -3, -5, 2, -1.5}, {"x", 7, 28, 1, 7, 4.0}, {"y", 8, 36, 1, 8, 4.5}, {"日本", 1, 9, 9, 9, 9.0}};
        bool ok = res.size() == 4;
        std::printf("result: [");
        for (size_t i = 0; i < res.size(); ++i) {
            const auto &v = res[i].second;
            const uint64_t n = v[0];
            const int64_t sum = vega::detail::from_bits<int64_t>(v[1]), lo = vega::detail::from_bits<int64_t>(v[2]),
                          hi = vega::detail::from_bits<int64_t>(v[3]);
            const double mean = vega::detail::from_bits<double>(v[4]);
            std::printf("%s(\"%s\", n=%llu, sum=%lld, min=%lld, max=%lld, mean=%g)", i ? ", " : "", res[i].first.c_str(),
                        (unsigned long long)n, (long long)sum, (long long)lo, (long long)hi, mean);
            if (i < 4) {
                const Want &w = want[i];
                ok = ok && res[i].first == w.k && n == w.n && sum == w.sum && lo == w.lo && hi == w.hi && mean == w.mean;
            }
        }
        std::printf("]\n%s\n", ok ? "ok" : "MISMATCH");
        return ok ? 0 : 1;
    } catch (const vega::Error &e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 2;
    }
}
