// fragment_distribution.h — FragmentLengthDistribution (mapper.hpp:83-139, mapper.cpp:5231-5333), the state behind the
// opaque gb_fragment_distribution handle.  The paired jobs and estimate() are in paired_job.cu.
#pragma once
#include "giraffe_b200.h"

#include <cstdint>
#include <set>

struct gb_fragment_distribution {
    std::multiset<double> lengths;
    bool is_fixed = false;
    double robust_estimation_fraction = 0.95;
    uint64_t maximum_sample_size = 1000, reestimation_frequency = 1000;
    double mu = 0.0, sigma = 1.0;

    // trimmed sample, then the method of moments for a normal truncated at +-a
    void estimate();
    void add(int64_t length) {
        if (is_fixed) return;
        lengths.insert((double)length);
        if (lengths.size() == maximum_sample_size) { estimate(); is_fixed = true; }
        else if (lengths.size() % reestimation_frequency == 0) estimate();
    }
};
