// emit_device.cu — gb_emit_gaf_device / gb_emit_gam_device / gb_emit_sam_device: GAF lines, GAM messages and SAM lines
// formatted on the GPU from records that are already in HBM.  The GAF / GAM format and record check are emit_format.h's, the
// code gb_emit_gaf / gb_emit_gam run on the host, so the bytes are those the host emitters write for the same records; the
// SAM line is sam_format.h's.  This file is the driver, one for the three formats.
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
#include "sam_format.h"

#include <cub/cub.cuh>

#include <algorithm>

namespace gb {
namespace {

constexpr uint32_t EMIT_BLOCK = 128;

// ---- formats --------------------------------------------------------------------------------------------------------
// What the driver asks of a format: n records, n_checks items to validate, whether record x is written, and its bytes
// over a sink.  FRAMED formats (GAM) add vg::io's group framing around each record's bytes.
struct GafFormat {
    static constexpr bool FRAMED = false;
    EmitArgs A;
    __host__ __device__ uint32_t n() const { return A.n; }
    __host__ __device__ uint32_t n_checks() const { return A.n > A.n_reads ? A.n : A.n_reads; }
    __device__ bool valid(uint32_t i) const { return (i >= A.n_reads || name_valid(A, i)) && (i >= A.n || record_valid(A, A.aln[i])); }
    __device__ bool present(uint32_t x) const { return !(A.aln[x].flags & GB_ALN_ABSENT); }
    template <class S> __device__ void body(S& s, uint32_t x) const { gaf_record(s, A, A.aln[x]); }
};
struct GamFormat : GafFormat {
    static constexpr bool FRAMED = true;
    template <class S> __device__ void body(S& s, uint32_t x) const { gam_message(s, A, A.aln[x]); }
};
struct SamFormat {
    static constexpr bool FRAMED = false;
    SamArgs A;
    __host__ __device__ uint32_t n() const { return A.n; }
    __host__ __device__ uint32_t n_checks() const { return A.n > A.n_reads ? A.n : A.n_reads; }
    __device__ bool valid(uint32_t i) const { return (i >= A.n_reads || sam_name_valid(A, i)) && (i >= A.n || sam_record_valid(A, A.rec[i])); }
    __device__ bool present(uint32_t x) const { return sam_present(A.rec[x]); }
    template <class S> __device__ void body(S& s, uint32_t x) const { sam_line(s, A, A.rec[x]); }
};

// ---- kernels --------------------------------------------------------------------------------------------------------
template <class F>
__global__ void emit_validate_kernel(F f, uint32_t* bad) {
    const uint32_t total = f.n_checks();
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x)
        if (!f.valid(i)) *bad = 1u;
}

// bytes[x] = the record's line (GAF, SAM) or message (GAM), 0 for a record that is not written; present[x] (GAM) = 1 for a
// written record.  Nothing is formatted when the batch was refused: the records may point anywhere.
template <class F>
__global__ void emit_size_kernel(F f, const uint32_t* bad, uint64_t* bytes, uint32_t* present) {
    const bool refused = *bad != 0;
    const uint32_t n = f.n();
    for (uint32_t x = blockIdx.x * blockDim.x + threadIdx.x; x <= n; x += gridDim.x * blockDim.x) {
        uint64_t sz = 0; uint32_t pr = 0;
        if (x < n && !refused && f.present(x)) {
            Count c;
            f.body(c, x);
            sz = c.n; pr = 1;
        }
        bytes[x] = sz;
        if (F::FRAMED) present[x] = pr;
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

template <class F>
__global__ void emit_fill_kernel(F f, const uint64_t* msg, const uint32_t* pidx, const uint64_t* off, char* out) {
    const uint32_t n = f.n();
    for (uint32_t x = blockIdx.x * blockDim.x + threadIdx.x; x < n; x += gridDim.x * blockDim.x) {
        if (!f.present(x)) continue;
        Write w{out + off[x]};
        if (F::FRAMED) {
            const uint32_t p = pidx[x];
            if (p % GAM_GROUP == 0) gam_header(w, min(GAM_GROUP, pidx[n] - p));
            varint(w, msg[x]);
        }
        f.body(w, x);
    }
}

// The driver: validate, size, scan, one wait for the total, fill.  `who` names the entry point in gb_last_error().
template <class F>
int emit_run(gb_device* d, const F& f, char* d_out, uint64_t out_cap, uint64_t* out_used, const char* who) {
    const uint32_t n = f.n();
    if (n == 0xffffffffu) return GB_ERR_ARG;                 // the scans run over n + 1 entries
    GB_CUDA(cudaSetDevice(d->device));
    constexpr bool GAM = F::FRAMED;

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
    const uint32_t vgrid = (uint32_t)std::min<uint64_t>(((uint64_t)f.n_checks() + EMIT_BLOCK) / EMIT_BLOCK, (uint64_t)d->n_sms * 64);
    GB_CUDA(cudaMemsetAsync(status, 0, 2 * sizeof(uint64_t), d->stream));
    emit_validate_kernel<<<vgrid, EMIT_BLOCK, 0, d->stream>>>(f, (uint32_t*)status);
    emit_size_kernel<<<grid, EMIT_BLOCK, 0, d->stream>>>(f, (const uint32_t*)status, bytes, present);
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
    if (h_status[0] & 0xffffffffull) { set_last_error(who, ": a record points outside its read, pools or the graph"); return GB_ERR_ARG; }
    const uint64_t total = h_status[1];
    *out_used = total;
    if (total > out_cap) { set_last_error(who, ": output capacity too small (*out_used holds the bytes needed)"); return GB_ERR_CAPACITY; }
    if (n) {
        emit_fill_kernel<<<grid, EMIT_BLOCK, 0, d->stream>>>(f, bytes, pidx, off, d_out);
        d->launches++;
        GB_CUDA(cudaGetLastError());
    }
    return GB_OK;
}

template <bool GAM>
int emit_device(gb_device* d, uint32_t n, const gb_alignment* d_aln, const gb_mapping* d_mappings, uint64_t mapping_pool_len,
                const uint32_t* d_edits, uint64_t edit_pool_len, uint32_t n_reads, const uint8_t* d_reads, const uint8_t* d_quals,
                const uint64_t* d_read_off, const uint8_t* d_names, const uint64_t* d_name_off, char* d_out, uint64_t out_cap, uint64_t* out_used) {
    if (!d || !d_aln || !d_reads || !d_read_off || !d_out || !out_used) return GB_ERR_ARG;
    EmitArgs A;
    A.n = n; A.aln = d_aln; A.maps = d_mappings; A.map_len = mapping_pool_len; A.edits = d_edits; A.edit_len = edit_pool_len;
    A.n_reads = n_reads; A.reads = d_reads; A.quals = d_quals; A.read_off = d_read_off; A.names = d_names; A.name_off = d_name_off;
    A.nodes = d->ix.nodes; A.seq = d->ix.seq; A.n_nodes = d->ix.n_nodes;
    if (GAM) return emit_run(d, GamFormat{A}, d_out, out_cap, out_used, "gb_emit_gam_device");
    return emit_run(d, GafFormat{A}, d_out, out_cap, out_used, "gb_emit_gaf_device");
}

int emit_sam_device(gb_device* d, uint32_t n, const gb_sam_record* d_rec, const uint32_t* d_cigar, uint64_t cigar_len,
                    uint32_t n_reads, const uint8_t* d_reads, const uint8_t* d_quals, const uint64_t* d_read_off,
                    const uint8_t* d_names, const uint64_t* d_name_off, char* d_out, uint64_t out_cap, uint64_t* out_used) {
    if (!d || !d_rec || !d_reads || !d_read_off || !d_out || !out_used) return GB_ERR_ARG;
    if (!d->ref_ready) { g_last_error = "gb_emit_sam_device: no reference paths on the handle (gb_device_set_ref_paths)"; return GB_ERR_ARG; }
    SamArgs A;
    A.n = n; A.rec = d_rec; A.cigar = d_cigar; A.cigar_len = cigar_len;
    A.n_reads = n_reads; A.reads = d_reads; A.quals = d_quals; A.read_off = d_read_off; A.names = d_names; A.name_off = d_name_off;
    A.n_paths = d->n_ref_paths; A.path_names = d->ref_names.ptr; A.path_name_off = d->ref_name_off.ptr;
    return emit_run(d, SamFormat{A}, d_out, out_cap, out_used, "gb_emit_sam_device");
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

extern "C" int gb_emit_sam_device(gb_device* dev, uint32_t n, const gb_sam_record* d_rec, const uint32_t* d_cigar, uint64_t cigar_len,
                                  uint32_t n_reads, const uint8_t* d_reads, const uint8_t* d_quals, const uint64_t* d_read_off,
                                  const uint8_t* d_names, const uint64_t* d_name_off, char* d_out, uint64_t out_cap, uint64_t* out_used) {
    return gb::guarded("gb_emit_sam_device", [&] { return gb::emit_sam_device(dev, n, d_rec, d_cigar, cigar_len, n_reads, d_reads, d_quals,
                                                                              d_read_off, d_names, d_name_off, d_out, out_cap, out_used); });
}
