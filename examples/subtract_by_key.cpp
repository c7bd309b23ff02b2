// subtract_by_key and semi_join (Spark's subtractByKey and left semi join; vega has neither), on integer and String keys:
//   events = (user, event id): (1,100) (2,200) (3,300) (1,101) (4,400) (2,201)   in 2 slices
//   banned = (2, 0) (4, 0) (9, 0)                                                  in 1 slice
//   active = (1, 7) (1, 8) (3, 7)                                                  in 2 slices
// events minus banned users keeps users 1 and 3; the semi join with active users keeps them too, each event once
// although user 1 is active twice.  The same with user names as String keys.  A key's rows keep the input order; the
// order of keys is unspecified, so the rows are sorted by key, stably.  Exit 0 only on the expected rows.
#include <algorithm>
#include <cstdio>
#include <string>

#include "vega_b200.hpp"

template <typename K>
static std::string show(const std::vector<std::pair<K, uint64_t>> &rows)
{
    std::string s;
    for (const auto &[k, v] : rows) {
        std::string ks;
        if constexpr (std::is_same_v<K, std::string>) ks = k; else ks = std::to_string(k);
        s += (s.empty() ? "" : ", ") + ("(" + ks + ", " + std::to_string(v) + ")");
    }
    return "[" + s + "]";
}

template <typename Rows>
static Rows by_key(Rows rows)
{
    std::stable_sort(rows.begin(), rows.end(), [](const auto &x, const auto &y) { return x.first < y.first; });
    return rows;
}

int main()
{
    try {
        auto sc = vega::Context::create();
        using Rows = std::vector<std::pair<uint64_t, uint64_t>>;
        auto events = sc->parallelize(Rows{{1, 100}, {2, 200}, {3, 300}, {1, 101}, {4, 400}, {2, 201}}, 2);
        auto banned = sc->parallelize(Rows{{2, 0}, {4, 0}, {9, 0}}, 1);
        auto active = sc->parallelize(Rows{{1, 7}, {1, 8}, {3, 7}}, 2);
        const Rows want = {{1, 100}, {1, 101}, {3, 300}};
        auto sub = by_key(events.subtract_by_key(banned, 3));
        auto semi = by_key(events.semi_join(active, 3));
        auto both = by_key(events.semi_join_n({active, banned}, 3, 0b01 << 1, 0b10 << 1));
        std::printf("subtract_by_key: %s\nsemi_join: %s\n", show(sub).c_str(), show(semi).c_str());

        using SRows = std::vector<std::pair<std::string, uint64_t>>;
        auto sevents = sc->parallelize(SRows{{"ann", 100}, {"bob", 200}, {"cy", 300}, {"ann", 101}, {"dee", 400}, {"bob", 201}}, 2);
        auto sbanned = sc->parallelize(SRows{{"bob", 0}, {"dee", 0}, {"zed", 0}}, 1);
        auto sactive = sc->parallelize(SRows{{"ann", 7}, {"ann", 8}, {"cy", 7}}, 2);
        const SRows swant = {{"ann", 100}, {"ann", 101}, {"cy", 300}};
        auto ssub = by_key(sevents.subtract_by_key(sbanned, 3));
        auto ssemi = by_key(sevents.semi_join(sactive, 3));
        std::printf("String subtract_by_key: %s\nString semi_join: %s\n", show(ssub).c_str(), show(ssemi).c_str());
        return sub == want && semi == want && both == want && ssub == swant && ssemi == swant ? 0 : 1;
    } catch (const vega::Error &e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 2;
    }
}
