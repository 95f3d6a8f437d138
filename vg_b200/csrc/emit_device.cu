// emit_device.cu — gb_emit_gaf_device / gb_emit_gam_device: GAF lines and GAM messages formatted on the GPU from records
// that are already in HBM.  The format and the record check are emit_format.h's, the code gb_emit_gaf / gb_emit_gam run on
// the host, so the bytes are those the host emitters write for the same records.  This file is the driver.
//
// Count / scan / fill, one thread per record:
//   validate   every record with record_valid and every name offset with name_valid, one flag for the whole batch
//   size       the exact bytes of each record over a Count sink (GAF: the line; GAM: the Alignment message)
//   scan       GAM: present records -> message index (group of 1000 and the place of its header); bytes -> offsets
//   fill       the bytes at the scanned offsets, the same formatter over a Write sink
// A thread formats its record straight into the output with byte stores; the lines are a few hundred bytes and the
// stores of a warp land in L2, which merges them before they reach HBM.
#include "giraffe_b200.h"
#include "device_state.cuh"
#include "emit_format.h"

#include <cub/cub.cuh>

#include <algorithm>

namespace gb {
namespace {

constexpr uint32_t EMIT_BLOCK = 128;

// ---- kernels --------------------------------------------------------------------------------------------------------
__global__ void emit_validate_kernel(EmitArgs A, uint32_t* bad) {
    const uint32_t total = max(A.n, A.n_reads);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        bool ok = true;
        if (i < A.n_reads && !name_valid(A, i)) ok = false;
        if (ok && i < A.n) ok = record_valid(A, A.aln[i]);
        if (!ok) *bad = 1u;
    }
}

// bytes[x] = the record's line (GAF) or message (GAM), 0 for an absent rank; present[x] (GAM) = 1 for a written record.
// Nothing is formatted when the batch was refused: the records may point anywhere.
template <bool GAM>
__global__ void emit_size_kernel(EmitArgs A, const uint32_t* bad, uint64_t* bytes, uint32_t* present) {
    const bool refused = *bad != 0;
    for (uint32_t x = blockIdx.x * blockDim.x + threadIdx.x; x <= A.n; x += gridDim.x * blockDim.x) {
        uint64_t sz = 0; uint32_t pr = 0;
        if (x < A.n && !refused) {
            const gb_alignment a = A.aln[x];
            if (!(a.flags & GB_ALN_ABSENT)) {
                Count c;
                if (GAM) gam_message(c, A, a); else gaf_record(c, A, a);
                sz = c.n; pr = 1;
            }
        }
        bytes[x] = sz;
        if (GAM) present[x] = pr;
    }
}

// GAM: a record's bytes in the stream = its group header when it opens a group + varint(message length) + message.
__global__ void gam_frame_kernel(uint32_t n, const uint64_t* msg, const uint32_t* pidx, uint64_t* framed) {
    const uint32_t np = pidx[n];
    for (uint32_t x = blockIdx.x * blockDim.x + threadIdx.x; x <= n; x += gridDim.x * blockDim.x) {
        uint64_t t = 0;
        if (x < n && pidx[x + 1] > pidx[x]) {
            const uint32_t p = pidx[x];
            t = varint_len(msg[x]) + msg[x];
            if (p % GAM_GROUP == 0) t += gam_header_len(min(GAM_GROUP, np - p));
        }
        framed[x] = t;
    }
}

template <bool GAM>
__global__ void emit_fill_kernel(EmitArgs A, const uint64_t* msg, const uint32_t* pidx, const uint64_t* off, char* out) {
    for (uint32_t x = blockIdx.x * blockDim.x + threadIdx.x; x < A.n; x += gridDim.x * blockDim.x) {
        const gb_alignment a = A.aln[x];
        if (a.flags & GB_ALN_ABSENT) continue;
        Write w{out + off[x]};
        if (GAM) {
            const uint32_t p = pidx[x];
            if (p % GAM_GROUP == 0) gam_header(w, min(GAM_GROUP, pidx[A.n] - p));
            varint(w, msg[x]);
            gam_message(w, A, a);
        } else {
            gaf_record(w, A, a);
        }
    }
}

template <bool GAM>
int emit_device(gb_device* d, uint32_t n, const gb_alignment* d_aln, const gb_mapping* d_mappings, uint64_t mapping_pool_len,
                const uint32_t* d_edits, uint64_t edit_pool_len, uint32_t n_reads, const uint8_t* d_reads, const uint8_t* d_quals,
                const uint64_t* d_read_off, const uint8_t* d_names, const uint64_t* d_name_off, char* d_out, uint64_t out_cap, uint64_t* out_used) {
    if (!d || !d_aln || !d_reads || !d_read_off || !d_out || !out_used) return GB_ERR_ARG;
    if (n == 0xffffffffu) return GB_ERR_ARG;                 // the scans run over n + 1 entries
    GB_CUDA(cudaSetDevice(d->device));
    EmitArgs A;
    A.n = n; A.aln = d_aln; A.maps = d_mappings; A.map_len = mapping_pool_len; A.edits = d_edits; A.edit_len = edit_pool_len;
    A.n_reads = n_reads; A.reads = d_reads; A.quals = d_quals; A.read_off = d_read_off; A.names = d_names; A.name_off = d_name_off;
    A.nodes = d->ix.nodes; A.seq = d->ix.seq; A.n_nodes = d->ix.n_nodes;

    // workspace: status {refused, total bytes}, bytes[n + 1], framed[n + 1] (GAM), off[n + 1], present / pidx[n + 1] (GAM), scan temp
    const size_t m = (size_t)n + 1;
    size_t scan64 = 0, scan32 = 0;
    GB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan64, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int64_t)m, d->stream));
    GB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan32, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int64_t)m, d->stream));
    size_t tb = std::max(scan64, scan32);
    uint64_t *status, *bytes, *framed, *off;
    uint32_t *present, *pidx;
    void* tmp;
    int rc = carve(d->emit_ws, [&](Carve& c) {
        status = c.take<uint64_t>(2); bytes = c.take<uint64_t>(m); framed = GAM ? c.take<uint64_t>(m) : bytes; off = c.take<uint64_t>(m);
        present = GAM ? c.take<uint32_t>(m) : nullptr; pidx = GAM ? c.take<uint32_t>(m) : nullptr; tmp = c.take<uint8_t>(tb);
    });
    if (rc) return rc;

    const uint32_t grid = (uint32_t)std::min<uint64_t>((m + EMIT_BLOCK - 1) / EMIT_BLOCK, (uint64_t)d->n_sms * 64);
    const uint32_t vgrid = (uint32_t)std::min<uint64_t>(((uint64_t)std::max(n, n_reads) + EMIT_BLOCK) / EMIT_BLOCK, (uint64_t)d->n_sms * 64);
    GB_CUDA(cudaMemsetAsync(status, 0, 2 * sizeof(uint64_t), d->stream));
    emit_validate_kernel<<<vgrid, EMIT_BLOCK, 0, d->stream>>>(A, (uint32_t*)status);
    emit_size_kernel<GAM><<<grid, EMIT_BLOCK, 0, d->stream>>>(A, (const uint32_t*)status, bytes, present);
    d->launches += 2;
    GB_CUDA(cudaGetLastError());
    if (GAM) {
        GB_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tb, present, pidx, (int64_t)m, d->stream));
        gam_frame_kernel<<<grid, EMIT_BLOCK, 0, d->stream>>>(n, bytes, pidx, framed);
        d->launches += 2;
        GB_CUDA(cudaGetLastError());
    }
    GB_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tb, framed, off, (int64_t)m, d->stream));
    d->launches++;
    GB_CUDA(cudaMemcpyAsync(status + 1, off + n, sizeof(uint64_t), cudaMemcpyDeviceToDevice, d->stream));
    uint64_t h_status[2];
    GB_CUDA(cudaMemcpyAsync(h_status, status, sizeof h_status, cudaMemcpyDeviceToHost, d->stream));
    GB_CUDA(cudaStreamSynchronize(d->stream));              // the one wait: the total decides whether the fill runs
    if (h_status[0] & 0xffffffffull) { g_last_error = GAM ? "gb_emit_gam_device: a record points outside its read, pools or the graph"
                                                          : "gb_emit_gaf_device: a record points outside its read, pools or the graph"; return GB_ERR_ARG; }
    const uint64_t total = h_status[1];
    *out_used = total;
    if (total > out_cap) { g_last_error = "gb_emit_*_device: output capacity too small (*out_used holds the bytes needed)"; return GB_ERR_CAPACITY; }
    if (n) {
        emit_fill_kernel<GAM><<<grid, EMIT_BLOCK, 0, d->stream>>>(A, bytes, pidx, off, d_out);
        d->launches++;
        GB_CUDA(cudaGetLastError());
    }
    return GB_OK;
}

} // namespace
} // namespace gb

#define GB_EMIT_DEVICE_ENTRY(NAME, GAM)                                                                                            \
    extern "C" int NAME(gb_device* dev, uint32_t n, const gb_alignment* d_aln, const gb_mapping* d_mappings, uint64_t mapping_pool_len, \
                        const uint32_t* d_edits, uint64_t edit_pool_len, uint32_t n_reads, const uint8_t* d_reads, const uint8_t* d_quals,  \
                        const uint64_t* d_read_off, const uint8_t* d_names, const uint64_t* d_name_off, char* d_out, uint64_t out_cap,        \
                        uint64_t* out_used) {                                                                                              \
        return gb::guarded(#NAME, [&] { return gb::emit_device<GAM>(dev, n, d_aln, d_mappings, mapping_pool_len, d_edits, edit_pool_len, n_reads, \
                                                                    d_reads, d_quals, d_read_off, d_names, d_name_off, d_out, out_cap, out_used); }); \
    }
GB_EMIT_DEVICE_ENTRY(gb_emit_gaf_device, false)
GB_EMIT_DEVICE_ENTRY(gb_emit_gam_device, true)
