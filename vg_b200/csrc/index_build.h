// index_build.h — the seam between the flat-index builder (index_builder.cpp), the GBZ reader (gbz_reader.cpp) and the
// device minimizer enumeration (index_device.cu).  Plain C++: every unit includes it.
#pragma once
#include "giraffe_b200.h"

#include <cstddef>
#include <cstdint>
#include <vector>

namespace gb {

// One minimizer occurrence of the table before placement: key, position (v << 10) | offset.
struct KeyPos { uint64_t key, pos; };

// What the window enumeration visited: start oriented nodes, continuations (strings whose minimizers were computed) and
// (key, position) pairs before de-duplication.
struct WindowCounts { uint64_t start_nodes = 0, continuations = 0, raw_pairs = 0; };

// gb_index_build_from_gbwt(_device): device < 0 builds on the host alone, device >= 0 enumerates the windows on that GPU.
int index_build_from_gbwt(int device, uint32_t n_node_ids, const uint8_t* node_seq, const uint64_t* node_off, uint32_t n_paths,
                          const uint32_t* gbwt_words, uint64_t n_words, const uint32_t* rec_off, const gb_dist_payload* dist,
                          uint32_t k, uint32_t w, uint64_t n_hits, const uint64_t* keys, const uint64_t* positions, gb_host_index** out);

// GB_OK when CUDA device `device` exists; GB_ERR_NO_DEVICE without a usable GPU, GB_ERR_ARG for an ordinal out of range.
int device_ready(int device);

// index_device.cu: the sorted, unique (key, position) pairs of every haplotype-consistent continuation of k + w - 2 bases
// behind every start node (forward_only: forward start nodes only), computed on GPU `device` from the builder's node
// records, both-orientation sequences and GBWT blob.  The same set the host window enumeration gives.
int window_pairs_device(int device, const std::vector<gb_node_rec>& nodes, const std::vector<uint8_t>& seq,
                        const std::vector<uint32_t>& gbwt, uint32_t k, uint32_t w, bool forward_only,
                        std::vector<KeyPos>& out, WindowCounts& counts);

} // namespace gb
