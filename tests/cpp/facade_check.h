// Shared by the facade examples: an EXPECT that counts failed expectations (a program exits 1 when any failed), and
// the raw file I/O through which they exchange arrays with their Python tests.
#pragma once
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "cupoch/cupoch_b200_facade.h"

inline int fails = 0;
#define EXPECT(cond)                                                          \
    do {                                                                      \
        if (!(cond)) { std::printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); ++fails; } \
    } while (0)

// the whole T elements of a file; empty when the file is missing
template <class T>
inline std::vector<T> read_file(const std::string &path) {
    std::vector<T> v;
    std::FILE *f = std::fopen(path.c_str(), "rb");
    if (!f) return v;
    T x;
    while (std::fread(&x, sizeof(T), 1, f) == 1) v.push_back(x);
    std::fclose(f);
    return v;
}

inline void write_file(const std::string &path, const void *data, size_t bytes) {
    std::FILE *f = std::fopen(path.c_str(), "wb");
    if (!f) {
        std::fprintf(stderr, "cannot write %s\n", path.c_str());
        std::exit(2);
    }
    if (bytes) std::fwrite(data, 1, bytes, f);
    std::fclose(f);
}

// [n][3] floats <-> n rows (a trailing partial row is dropped)
inline std::vector<Eigen::Vector3f> rows3(const std::vector<float> &flat) {
    std::vector<Eigen::Vector3f> rows;
    for (size_t i = 0; i + 2 < flat.size(); i += 3) rows.push_back(Eigen::Vector3f(flat[i], flat[i + 1], flat[i + 2]));
    return rows;
}

inline std::vector<float> rows3(const std::vector<Eigen::Vector3f> &rows) {
    std::vector<float> flat;
    for (const auto &r : rows) flat.insert(flat.end(), {r[0], r[1], r[2]});
    return flat;
}
