// The textbook combine_by_key example: a per-key average, here with the (sum, count) combiner replaced by the named
// MEAN aggregate, next to the COUNT and MAX of the same key, all from one shuffle.  Expected output (sorted by key):
//   result: [(120, n=7, mean=4, max=7), (121, n=8, mean=4.5, max=8)]
#include <algorithm>
#include <cstdio>

#include "vega_b200.hpp"

int main()
{
    try {
        auto sc = vega::Context::create();
        std::vector<std::pair<uint64_t, int64_t>> vec;
        for (int i = 1; i <= 7; ++i) vec.emplace_back('x', i);
        for (int i = 1; i <= 8; ++i) vec.emplace_back('y', i);
        auto r = sc->make_rdd(vec, 4);
        auto res = r.combine_by_key({VB_AGG_COUNT, VB_AGG_MEAN, VB_AGG_MAX}, 4);
        std::sort(res.begin(), res.end());
        std::printf("result: [");
        bool ok = res.size() == 2;
        for (size_t i = 0; i < res.size(); ++i) {
            const uint64_t n = res[i].second[0];
            const double mean = vega::detail::from_bits<double>(res[i].second[1]);
            const int64_t hi = vega::detail::from_bits<int64_t>(res[i].second[2]);
            std::printf("%s(%llu, n=%llu, mean=%g, max=%lld)", i ? ", " : "", (unsigned long long)res[i].first, (unsigned long long)n, mean,
                        (long long)hi);
            ok = ok && n == (i ? 8u : 7u) && mean == (i ? 4.5 : 4.0) && hi == (i ? 8 : 7);
        }
        std::printf("]\n");
        return ok ? 0 : 1;
    } catch (const vega::Error &e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 2;
    }
}
