// SegmentPlane's sampler run by thrust itself: the toolkit's thrust headers compiled for the CPP backend with g++.
// random_functor and the tabulate / sort_by_key chain are written exactly as the reference's sampling loop
// (segmentation.cu:38-48, 214-229) writes them, minus __device__.
//   thrust_ransac_pin OUT N seed...   writes, per seed, the N keys and d_cards[0..2] after that seed's sort (int32)
#include <thrust/host_vector.h>
#include <thrust/random.h>
#include <thrust/sequence.h>
#include <thrust/sort.h>
#include <thrust/tabulate.h>

#include <cstdio>
#include <cstdlib>

struct random_functor {
    random_functor(int seed, int n) : seed_(seed), n_(n) {}
    const int seed_;
    const int n_;
    int operator()(size_t idx) const {
        thrust::default_random_engine eng(seed_);
        thrust::uniform_int_distribution<int> dist(0, n_ - 1);
        eng.discard(idx);
        return dist(eng);
    }
};

int main(int argc, char **argv) {
    if (argc < 3) return 2;
    FILE *f = std::fopen(argv[1], "wb");
    if (!f) return 1;
    const int n = std::atoi(argv[2]);
    thrust::host_vector<int> d_cards(n), d_keys(n);
    thrust::sequence(d_cards.begin(), d_cards.end());
    for (int a = 3; a < argc; ++a) {
        thrust::tabulate(d_keys.begin(), d_keys.end(), random_functor((int)std::strtol(argv[a], nullptr, 10), n));
        std::fwrite(d_keys.data(), sizeof(int), n, f);
        thrust::sort_by_key(d_keys.begin(), d_keys.end(), d_cards.begin());
        std::fwrite(d_cards.data(), sizeof(int), 3, f);
    }
    std::fclose(f);
    return 0;
}
