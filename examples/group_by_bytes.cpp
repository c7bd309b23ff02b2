// The reference's examples/group_by.rs with byte-slice keys b"x" and b"y" (Rust Vec<u8>, placed by the slice hash:
// MetroHash64_1(le64(len) ‖ bytes) % n).  Expected output (the order of keys is unspecified; sorted here):
//   result: [("x", [1, 2, 3, 4, 5, 6, 7]), ("y", [1, 2, 3, 4, 5, 6, 7, 8])]
#include <algorithm>
#include <cstdio>

#include "vega_b200.hpp"

int main()
{
    try {
        auto sc = vega::Context::create();
        const std::vector<uint8_t> x{'x'}, y{'y'};
        std::vector<std::pair<std::vector<uint8_t>, int64_t>> vec;
        for (int i = 1; i <= 7; ++i) vec.emplace_back(x, i);
        for (int i = 1; i <= 8; ++i) vec.emplace_back(y, i);
        const uint32_t n_splits = 4;
        auto res = sc->make_rdd(vec, 4).group_by_key(n_splits);
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
        // count_by_value over Vec<u8> items
        auto counts = sc->parallelize(std::vector<std::vector<uint8_t>>{x, y, x}, 2).count_by_value();
        std::sort(counts.begin(), counts.end());
        ok = ok && counts.size() == 2 && counts[0] == std::make_pair(std::string("x"), (uint64_t)2) &&
             counts[1] == std::make_pair(std::string("y"), (uint64_t)1);
        return ok ? 0 : 1;
    } catch (const vega::Error &e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 2;
    }
}
