// entity_list.cu -- bgs_entity_list's device side: the per-frame expansion of the list's compact records into the segment
// table bgs_render_entities_many's kernels read, and the edits' scatters of records and transforms.
#include "launch.cuh"

namespace bgs {
namespace {

constexpr int EXPAND_THREADS = 128;   // 128 segments of 344 B staged in shared memory (43 KB)
constexpr int SCATTER_THREADS = 256;

// Segment j from record j and the frame's view: each thread builds its segment in shared memory, then the CTA stores its
// run of segments with coalesced 8-byte stores.
__global__ void __launch_bounds__(EXPAND_THREADS)
entity_list_expand_kernel(const EntityRec* __restrict__ recs, const uint32_t* __restrict__ offset, uint32_t k, bgs_view view,
                          uint32_t radix_sort_depth_bits, uint32_t n_total, SceneSeg* __restrict__ seg) {
    static_assert(sizeof(SceneSeg) % 8 == 0, "segments are stored in 8-byte words");
    __shared__ SceneSeg s[EXPAND_THREADS];
    const uint32_t base = blockIdx.x * EXPAND_THREADS;
    const uint32_t j = base + threadIdx.x;
    if (j < k) {
        const EntityRec& r = recs[j];
        SceneSeg& o = s[threadIdx.x];
        o.fc = make_frame_consts(view, r.uni, radix_sort_depth_bits, r.gaussian_mode, r.rasterize_mode, r.aabb, r.adaptive,
                                 r.draw_mode, n_total, r.cov_pre, 0u);
        o.pos = r.pos;
        o.blocks = r.blocks;
        o.offset = offset[j];
        o.n = r.n;
        o.group = r.group;
    }
    __syncthreads();
    const uint32_t words = min((uint32_t)EXPAND_THREADS, k - base) * (uint32_t)(sizeof(SceneSeg) / 8);
    const uint2* src = reinterpret_cast<const uint2*>(s);
    uint2* dst = reinterpret_cast<uint2*>(seg + base);
    for (uint32_t w = threadIdx.x; w < words; w += EXPAND_THREADS) dst[w] = src[w];
}

// entities idx[i] (distinct) take record i and its table entries
__global__ void __launch_bounds__(SCATTER_THREADS)
entity_list_scatter_kernel(EntityListUpload u, uint32_t count, EntityListArrays a) {
    const uint32_t i = blockIdx.x * SCATTER_THREADS + threadIdx.x;
    if (i >= count) return;
    const uint32_t j = u.idx[i];
    a.recs[j] = u.recs[i];
    a.offset[j] = u.offset[i];
    a.times[j] = u.times[i];
    a.classes[j] = u.classes[i];
    a.kinds[j] = u.kinds[i];
    a.kinds_box[j] = u.kinds[i] | BOX_KIND;
}

// count row-major 4x4 matrices into the column-major transforms of records dst[0 .. count): one thread per element
__global__ void __launch_bounds__(SCATTER_THREADS)
entity_list_transforms_kernel(const float* __restrict__ m, uint32_t count, EntityRec* __restrict__ dst) {
    const uint32_t t = blockIdx.x * SCATTER_THREADS + threadIdx.x;
    const uint32_t i = t >> 4, e = t & 15u;   // e = column * 4 + row
    if (i >= count) return;
    dst[i].uni.transform[e] = m[(size_t)i * 16 + (e & 3u) * 4 + (e >> 2)];
}

}  // namespace

cudaError_t launch_entity_list_expand(const EntityRec* recs, const uint32_t* offset, uint32_t k, const bgs_view& view,
                                      uint32_t radix_sort_depth_bits, uint32_t n_total, SceneSeg* seg, cudaStream_t stream) {
    entity_list_expand_kernel<<<(k + EXPAND_THREADS - 1) / EXPAND_THREADS, EXPAND_THREADS, 0, stream>>>(
        recs, offset, k, view, radix_sort_depth_bits, n_total, seg);
    return cudaGetLastError();
}

cudaError_t launch_entity_list_scatter(const EntityListUpload& u, uint32_t count, const EntityListArrays& a, cudaStream_t stream) {
    entity_list_scatter_kernel<<<(count + SCATTER_THREADS - 1) / SCATTER_THREADS, SCATTER_THREADS, 0, stream>>>(u, count, a);
    return cudaGetLastError();
}

cudaError_t launch_entity_list_transforms(const float* m, uint32_t count, EntityRec* dst, cudaStream_t stream) {
    const uint64_t threads = (uint64_t)count * 16;
    entity_list_transforms_kernel<<<(unsigned)((threads + SCATTER_THREADS - 1) / SCATTER_THREADS), SCATTER_THREADS, 0, stream>>>(
        m, count, dst);
    return cudaGetLastError();
}

}  // namespace bgs
