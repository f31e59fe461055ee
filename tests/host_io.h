// The stdin / stdout protocol of the host harnesses (tests/host_exe.py: hexes, run, floats): numbers are read as C hex
// floats, "inf" or "nan" and printed as hex floats, NaN as "nan".
#pragma once

#include <cstdio>
#include <cstdlib>
#include <vector>

static inline double rd()
{
    char buf[64];
    if (scanf("%63s", buf) != 1) exit(2);
    return strtod(buf, nullptr);
}
static inline long long rl() { return (long long)rd(); }
static inline void pr(double x)
{
    if (x != x) printf(" nan");
    else printf(" %a", x);
}
static inline std::vector<double> rv(size_t n)
{
    std::vector<double> v(n);
    for (auto &x : v) x = rd();
    return v;
}
