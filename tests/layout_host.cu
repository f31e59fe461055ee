// CPU exercise of Layout (csrc/entry.h), the one rule that places the regions of every entry point's scratch.
// Built and run by tests/test_layout_cpu.py (nvcc for the host, no GPU).
//   usage: layout_host <at> <bytes>...  -> the regions' offsets on one line, the layout's bytes() on the next; exit status
//   1 when Layout::at does not point at base + offset
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "../pyaudioanalysis_b200/csrc/entry.h"

int main(int argc, char **argv)
{
    if (argc < 2) return 2;
    Layout L(std::strtoull(argv[1], nullptr, 10));
    std::vector<size_t> at;
    for (int i = 2; i < argc; ++i) at.push_back(L.add(std::strtoull(argv[i], nullptr, 10)));
    std::vector<char> block(L.bytes() + 1);
    char *base = block.data();
    for (size_t i = 0; i < at.size(); ++i) {
        if (reinterpret_cast<char *>(Layout::at<double>(base, at[i])) != base + at[i]) return 1;
        std::printf("%s%zu", i ? " " : "", at[i]);
    }
    std::printf("\n%zu\n", L.bytes());
    return 0;
}
