// Sessions from sorted value lists: group_by_key(num_splits, sorted_values = true) gives each user's event times in
// ascending order, sorted on the device, so a session split needs no sort on the host.  A gap of more than 30 time
// units starts a new session.  The same join with sorted_values gives a key's rows in ascending (v, w) order.
// Expected output:
//   user 7: sessions [[3, 5, 20], [90, 95]]
//   user 9: sessions [[-4, 1], [40]]
//   join 7: (3, 100) (3, 200) (5, 100) (5, 200) ...
#include <algorithm>
#include <cstdio>

#include "vega_b200.hpp"

int main()
{
    try {
        auto sc = vega::Context::create();
        std::vector<std::pair<uint64_t, int64_t>> events = {{7, 90}, {9, 40}, {7, 3}, {9, 1}, {7, 20}, {7, 95}, {9, -4}, {7, 5}};
        auto res = sc->make_rdd(events, 3).group_by_key(2, true);
        std::sort(res.begin(), res.end());
        bool ok = res.size() == 2;
        const std::vector<std::vector<std::vector<int64_t>>> want = {{{3, 5, 20}, {90, 95}}, {{-4, 1}, {40}}};
        for (size_t u = 0; u < res.size(); ++u) {
            std::vector<std::vector<int64_t>> sessions;
            for (size_t i = 0; i < res[u].second.size(); ++i) {
                const int64_t t = res[u].second[i];
                if (i == 0 || t - res[u].second[i - 1] > 30) sessions.emplace_back();
                sessions.back().push_back(t);
            }
            std::printf("user %llu: sessions [", (unsigned long long)res[u].first);
            for (size_t s = 0; s < sessions.size(); ++s) {
                std::printf("%s[", s ? ", " : "");
                for (size_t i = 0; i < sessions[s].size(); ++i) std::printf("%s%lld", i ? ", " : "", (long long)sessions[s][i]);
                std::printf("]");
            }
            std::printf("]\n");
            ok = ok && u < want.size() && sessions == want[u];
        }
        std::vector<std::pair<uint64_t, int64_t>> tags = {{7, 200}, {7, 100}};
        auto rows = sc->make_rdd(events, 2).join(sc->make_rdd(tags, 1), 2, true);
        std::printf("join 7:");
        std::vector<std::pair<int64_t, int64_t>> got;
        for (auto &r : rows) {
            std::printf(" (%lld, %lld)", (long long)r.second.first, (long long)r.second.second);
            got.push_back(r.second);
        }
        std::printf("\n");
        ok = ok && got.size() == 10 && std::is_sorted(got.begin(), got.end());
        return ok ? 0 : 1;
    } catch (const vega::Error &e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 2;
    }
}
