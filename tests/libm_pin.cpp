// tests/libm_pin.cpp -- TEST INFRASTRUCTURE: pins the device's libm restatements (pbrt-v3-distributed_b200/csrc, compiled
// here as plain C++) against the host libm -- the calls the reference makes -- bit for bit (both NaN also passes):
//   pt_expf / pt_logf / pt_atanf   every float bit pattern            std::exp / std::log / std::atan (float)
//   pt_sinf / pt_cosf              every float with |x| < 8            std::sin / std::cos (float)
//   pt_acosf                       every float in [-1, 1]              std::acos (float)
//   pt_atan2f                      2*10^8 random pairs + edge pairs    std::atan2 (float)
//   pt_cos / pt_sin (double)       every phi tr_sample11 can form      ::cos / ::sin (double)
//   g++ -O2 -std=c++17 -ffp-contract=off -fno-builtin-sin -fno-builtin-cos -pthread tests/libm_pin.cpp -o /tmp/libm_pin
//   /tmp/libm_pin [stride]     (stride 1 = exhaustive, about a minute on 8 cores; a larger stride checks every stride-th input)
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <functional>
#include <thread>
#include <vector>

#include "../pbrt-v3-distributed_b200/csrc/pt_sphere.cuh"

using namespace b200pt;

static uint64_t stride = 1;
static bool any_fail = false;

static bool same32(float a, float b) { return float_as_uint(a) == float_as_uint(b) || (std::isnan(a) && std::isnan(b)); }
static bool same64(double a, double b) { return double_as_u64(a) == double_as_u64(b) || (std::isnan(a) && std::isnan(b)); }

// Counts the inputs k in [0, n) (every stride-th) for which ok(k) is false; prints the count and the smallest such k.
static void pin(const char *name, uint64_t n, const std::function<bool(uint64_t)> &ok, const char *what) {
    const unsigned nt = std::max(1u, std::thread::hardware_concurrency());
    std::atomic<uint64_t> bad{0}, first{~0ull};
    std::vector<std::thread> pool;
    for (unsigned t = 0; t < nt; ++t)
        pool.emplace_back([&, t]() {
            uint64_t b = 0;
            for (uint64_t k = t * stride; k < n; k += nt * stride)
                if (!ok(k)) {
                    ++b;
                    uint64_t cur = first.load();
                    while (k < cur && !first.compare_exchange_weak(cur, k)) {
                    }
                }
            bad += b;
        });
    for (auto &th : pool) th.join();
    printf("%s: %llu mismatches", name, (unsigned long long)bad.load());
    if (bad) printf(" (first at %s 0x%llx)", what, (unsigned long long)first.load());
    printf("\n");
    any_fail |= bad != 0;
}

// |x| < lim: k -> +-(bits k / 2), so that k covers both signs
static float signed_float(uint64_t k) { return uint_as_float((uint32_t)(k >> 1) | (k & 1 ? 0x80000000u : 0u)); }

static uint64_t splitmix64(uint64_t z) {
    z += 0x9e3779b97f4a7c15ull;
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}

int main(int argc, char **argv) {
    stride = argc > 1 ? (uint64_t)atoll(argv[1]) : 1;
    const uint64_t all = 1ull << 32;
    pin("expf", all, [](uint64_t k) { const float x = uint_as_float((uint32_t)k); return same32(std::exp(x), pt_expf(x)); }, "bits");
    pin("logf", all, [](uint64_t k) { const float x = uint_as_float((uint32_t)k); return same32(std::log(x), pt_logf(x)); }, "bits");
    pin("atanf", all, [](uint64_t k) { const float x = uint_as_float((uint32_t)k); return same32(std::atan(x), pt_atanf(x)); }, "bits");
    const uint64_t below8 = 2ull * float_as_uint(8.f);
    pin("sinf", below8, [](uint64_t k) { const float x = signed_float(k); return same32(std::sin(x), pt_sinf(x)); }, "2*bits+sign");
    pin("cosf", below8, [](uint64_t k) { const float x = signed_float(k); return same32(std::cos(x), pt_cosf(x)); }, "2*bits+sign");
    pin("acosf", 2ull * (float_as_uint(1.f) + 1),
        [](uint64_t k) { const float x = signed_float(k); return same32(std::acos(x), pt_acosf(x)); }, "2*bits+sign");
    // atan2f: even pairs any two bit patterns, odd pairs two floats in [-3, 3) ...
    pin("atan2f random", 200000000ull, [](uint64_t k) {
        const uint64_t h = splitmix64(k);
        float y = uint_as_float((uint32_t)h), x = uint_as_float((uint32_t)(h >> 32));
        if (k & 1) {
            y = (float)(h & 0xffffffu) * 0x1p-24f * 6.f - 3.f;
            x = (float)((h >> 32) & 0xffffffu) * 0x1p-24f * 6.f - 3.f;
        }
        return same32(std::atan2(y, x), pt_atan2f(y, x));
    }, "pair");
    // ... and edge pairs: +-0, +-inf, NaN, subnormals, y = +-x and |y / x| = 2^+-30, 2^+-60, 2^+-61 (with neighbours)
    static const float edge[] = {0.f, -0.f, INFINITY, -INFINITY, NAN, 1.f, -1.f, 0.5f, 3.f, -7.25f, 1e-30f, 1e30f,
                                 0x1p-149f, -0x1p-149f, 0x1p-130f, -0x1p-130f, 0x1p-126f, 0x1.fffffep127f};
    const uint64_t ne = sizeof(edge) / sizeof(edge[0]);
    const uint64_t saved = stride;
    stride = 1;
    pin("atan2f edges", ne * ne, [&](uint64_t k) {
        const float y = edge[k / ne], x = edge[k % ne];
        return same32(std::atan2(y, x), pt_atan2f(y, x));
    }, "pair");
    pin("atan2f ratios", 1ull << 20, [](uint64_t k) {
        static const int e[] = {0, 30, -30, 60, -60, 61, -61, 0};
        const float x = uint_as_float((uint32_t)(splitmix64(k >> 6) & 0x807fffffu) | 0x3f800000u);  // +-[1, 2)
        const float s = (k >> 3) & 1 ? -1.f : 1.f;
        float y = s * std::ldexp(x, e[k & 7]);
        const int nb = (int)((k >> 4) & 3);
        if (nb == 1) y = std::nextafter(y, INFINITY);
        if (nb == 2) y = std::nextafter(y, -INFINITY);
        return same32(std::atan2(y, x), pt_atan2f(y, x));
    }, "case");
    stride = saved;
    // tr_sample11's normal-incidence branch: phi = (float)(6.28318530718 * (double)U2) for every float U2 in [0, 1)
    const uint64_t nU2 = float_as_uint(1.f);
    pin("cos(double phi)", nU2, [](uint64_t k) {
        const double phi = (float)(6.28318530718 * (double)uint_as_float((uint32_t)k));
        return same64(::cos(phi), pt_cos(phi));
    }, "U2 bits");
    pin("sin(double phi)", nU2, [](uint64_t k) {
        const double phi = (float)(6.28318530718 * (double)uint_as_float((uint32_t)k));
        return same64(::sin(phi), pt_sin(phi));
    }, "U2 bits");
    printf("%s over %s\n", any_fail ? "FAIL" : "OK", stride == 1 ? "every input" : "a strided subset of the inputs");
    return any_fail ? 1 : 0;
}
