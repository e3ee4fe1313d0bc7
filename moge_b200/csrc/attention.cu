// Multi-head self-attention of the DINOv2 blocks (reference: dinov2/layers/attention.py:70-81, SDPA with
// scale hd^-0.5, no mask) as one wgmma kernel: S = Q K^T from shared memory, single-pass online softmax in registers,
// O~ += P V with P taken straight from the registers that held S (the fp32 accumulator fragment of S is, after packing to
// 16 bit, the A-operand fragment of the P V MMA), O accumulated in registers.
//
// Layout: qkv is the QKV-GEMM output [rows, 3*D] (16-bit), the token rows of all images PACKED back to back (images may have
// different token counts: ragged batches); Q/K/V tiles of head h are the column windows [h*64, D+h*64, 2D+h*64) fetched by
// TMA straight from that buffer (no head-major repack): Q and K tiles are K-major wgmma operands, the V tile ([kv][hd], hd
// contiguous) is consumed as an MN-major B operand.  A K/V box that runs past the image's last token reads the next image's
// rows (or TMA zero fill past the buffer): those columns are masked to -inf before the softmax.
// Output: out[row0 + q, h*64 + d] (16-bit), the A operand of the projection GEMM.
//
// PERSISTENT: one CTA per SM walks a contiguous range of work items (image, head, pair of 128-row query tiles) from a host-built
// list (cost-balanced ranges, consecutive query tiles of one (image, head) on the same SM -> K/V come from L2).  Warpgroup 0
// streams Q and the K/V ring by TMA; consumer warpgroup g (1 + g) owns query tile g of the item and runs it as two 64-row
// halves, each with its own O accumulator and running max / sum.
#include "common.cuh"
#include "host_api.h"
#include <vector>

namespace mg {

constexpr int ATT_HD = 64;
constexpr int ATT_BQ = 128;       // query rows per consumer warpgroup
constexpr int ATT_BKV = 128;      // keys per tile
constexpr int ATT_KV_STAGES = 5;
constexpr int ATT_TILE_BYTES = 128 * 128;   // [128 rows][64 x 16-bit]
constexpr int ATT_THREADS = 128 + 256;   // warpgroup 0: TMA; warpgroups 1, 2: MMA + softmax
// smem: Q0,Q1 | K[stages] | V[stages] | barriers
constexpr int ATT_SMEM = (2 + 2 * ATT_KV_STAGES) * ATT_TILE_BYTES + 1024 + 256;
static_assert(ATT_SMEM <= kMaxDynSmem, "attention_kernel: Q + K/V ring exceed the shared memory of one CTA");
static_assert((2 + 4 * ATT_KV_STAGES) * 8 <= 256, "attention_kernel: barrier block overflows its 256 bytes");

struct AttnParams {
    void* out;               // [rows, D] 16-bit
    const AttnItem* items;   // work list (device)
    const int2* ranges;      // per CTA: [begin, end) into items
    int D;
    float scale_log2;        // hd^-0.5 * log2(e)
};

template <bool BF16>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attention_kernel(const __grid_constant__ CUtensorMap mapQKV, const AttnParams p) {
    pdl_launch_dependents();      // (the wait sits after the barrier set-up below: that prologue overlaps the previous kernel's tail)
    using H = H16<BF16>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    constexpr int ST = ATT_KV_STAGES;
    uint8_t* sQ = smem;                                        // 2 tiles
    uint8_t* sK = sQ + 2 * ATT_TILE_BYTES;
    uint8_t* sV = sK + ST * ATT_TILE_BYTES;
    uint64_t* bars = reinterpret_cast<uint64_t*>(sV + ST * ATT_TILE_BYTES);
    uint64_t* q_full = bars;                 // 1: Q tiles of the current item landed
    uint64_t* q_empty = bars + 1;            // every S MMA of the current item has completed -> the next item's Q may be loaded
    uint64_t* k_full = bars + 2;
    uint64_t* k_empty = k_full + ST;
    uint64_t* v_full = k_empty + ST;
    uint64_t* v_empty = v_full + ST;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int2 rng = p.ranges[blockIdx.x];

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&mapQKV);
        // empty barriers: one arrival per consumer warp (8) once its warpgroup's MMAs reading the buffer have completed
        mbar_init(q_full, 1); mbar_init(q_empty, 8);
        for (int s = 0; s < ST; ++s) {
            mbar_init(&k_full[s], 1); mbar_init(&k_empty[s], 8);
            mbar_init(&v_full[s], 1); mbar_init(&v_empty[s], 8);
        }
        fence_mbar_init();
    }
    __syncthreads();
    pdl_wait();

    if (warp < 4) {
        // ========================================================== TMA producer (warp 0, converged, one elected lane issues)
        regs_dec<40>();
        if (warp != 0) return;
        int s = 0; uint32_t ph = 0;
        for (int it = rng.x; it < rng.y; ++it) {
            const AttnItem item = p.items[it];
            const int li = it - rng.x;
            const int nkv = (item.n + ATT_BKV - 1) / ATT_BKV;
            if (li > 0) mbar_wait(q_empty, (li - 1) & 1);
            if (elect_one()) {
                // both query tiles always: the second one of an image's last item may lie past the image (its rows are computed and
                // not stored), so that every consumer warpgroup walks every K/V stage
                mbar_arrive_expect_tx(q_full, 2 * ATT_TILE_BYTES);
                tma_load_2d(sQ, &mapQKV, q_full, item.head * ATT_HD, item.row0 + item.q0);
                tma_load_2d(sQ + ATT_TILE_BYTES, &mapQKV, q_full, item.head * ATT_HD, item.row0 + item.q0 + ATT_BQ);
            }
            __syncwarp();
            for (int j = 0; j < nkv; ++j) {
                mbar_wait(&k_empty[s], ph ^ 1);
                if (elect_one()) {
                    mbar_arrive_expect_tx(&k_full[s], ATT_TILE_BYTES);
                    tma_load_2d(sK + s * ATT_TILE_BYTES, &mapQKV, &k_full[s], p.D + item.head * ATT_HD, item.row0 + j * ATT_BKV);
                }
                __syncwarp();
                mbar_wait(&v_empty[s], ph ^ 1);
                if (elect_one()) {
                    mbar_arrive_expect_tx(&v_full[s], ATT_TILE_BYTES);
                    tma_load_2d(sV + s * ATT_TILE_BYTES, &mapQKV, &v_full[s], 2 * p.D + item.head * ATT_HD, item.row0 + j * ATT_BKV);
                }
                __syncwarp();
                if (++s == ST) { s = 0; ph ^= 1; }
            }
        }
        return;
    }
    // ============================================================== consumers: S = Q K^T, softmax, O += P V, normalise + store
    regs_inc<232>();
    const int g = (warp - 4) >> 2;          // query tile of the item
    const int wl = warp & 3;
    const float sc = p.scale_log2;
    // accumulator fragment: this thread's rows r0 and r0 + 8 of a 64-row half; columns 8 (i / 4) + 2 (lane % 4) + i % 2
    const int r0 = 16 * wl + (lane >> 2);
    const int cq = 2 * (lane & 3);
    int s = 0; uint32_t ph = 0;
    for (int it = rng.x; it < rng.y; ++it) {
        const AttnItem item = p.items[it];
        const int li = it - rng.x;
        const int nkv = (item.n + ATT_BKV - 1) / ATT_BKV;
        mbar_wait(q_full, li & 1);
        float o[2][32];
        float m[2][2], l[2][2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int i = 0; i < 32; ++i) o[h][i] = 0.f;
            m[h][0] = m[h][1] = -INFINITY;
            l[h][0] = l[h][1] = 0.f;
        }
        for (int j = 0; j < nkv; ++j) {
            const int kv_left = item.n - j * ATT_BKV;
            mbar_wait(&k_full[s], ph);
            mbar_wait(&v_full[s], ph);
            const uint32_t kaddr = smem_u32(sK + s * ATT_TILE_BYTES);
            const uint32_t vaddr = smem_u32(sV + s * ATT_TILE_BYTES);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float sv[64];
#pragma unroll
                for (int i = 0; i < 64; ++i) sv[i] = 0.f;
                wgmma_fence();
                const uint64_t qd = make_sdesc_sw128(smem_u32(sQ + g * ATT_TILE_BYTES + h * 64 * 128));
                const uint64_t kd = make_sdesc_sw128(kaddr);
#pragma unroll
                for (int k = 0; k < ATT_HD / 16; ++k) Wgmma<ATT_BKV, BF16>::ss(sv, qd + 2 * k, kd + 2 * k, 1u);
                wgmma_commit();
                wgmma_wait<0>();
                reg_fence(sv);
                if (kv_left < ATT_BKV) {                    // only the last tile has padding columns
#pragma unroll
                    for (int i = 0; i < 64; ++i)
                        if (8 * (i >> 2) + cq + (i & 1) >= kv_left) sv[i] = -INFINITY;
                }
                // row max over the quad of lanes sharing a row
                float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
                for (int i = 0; i < 64; ++i) mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], sv[i]);
                float alpha[2], mb[2];
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
                    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
                    const float m_new = fmaxf(m[h][r], mx[r]);
                    alpha[r] = ex2_approx((m[h][r] - m_new) * sc);        // 0 on the first tile (m = -inf)
                    m[h][r] = m_new;
                    mb[r] = m_new * sc;
                    l[h][r] *= alpha[r];
                }
#pragma unroll
                for (int i = 0; i < 32; ++i) o[h][i] *= alpha[(i >> 1) & 1];
                // P = 2^(S sc - m sc), packed to 16 bit in the A-operand fragment order of the P V MMA (k-step kk: columns 16 kk ..)
                uint32_t pa[32];
#pragma unroll
                for (int i = 0; i < 64; i += 2) {
                    const int r = (i >> 1) & 1;
                    const float e0 = ex2_approx(fmaf(sv[i], sc, -mb[r])), e1 = ex2_approx(fmaf(sv[i + 1], sc, -mb[r]));
                    l[h][r] += e0 + e1;
                    pa[i >> 1] = H::pack(e0, e1);
                }
                wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < ATT_BKV / 16; ++kk) {
                    // B: V tile [kv][hd], MN-major, 16 kv rows (= 2 groups of 8 x 128 B) per K-step
                    const uint64_t vd = make_sdesc_sw128(vaddr + kk * 16 * 128, /*lbo=*/ATT_TILE_BYTES, /*sbo=*/1024);
                    wgmma_rs_n64_tb<BF16>(o[h], pa + 4 * kk, vd, 1u);
                }
                wgmma_commit();
                wgmma_wait<0>();
                reg_fence(o[h]);
            }
            __syncwarp();
            if (lane == 0) { mbar_arrive(&k_empty[s]); mbar_arrive(&v_empty[s]); }
            if (++s == ST) { s = 0; ph ^= 1; }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(q_empty);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                l[h][r] += __shfl_xor_sync(0xffffffffu, l[h][r], 1);
                l[h][r] += __shfl_xor_sync(0xffffffffu, l[h][r], 2);
            }
            const float inv[2] = {1.0f / l[h][0], 1.0f / l[h][1]};
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const int qrow = item.q0 + g * ATT_BQ + h * 64 + r0 + 8 * r;
                if (qrow >= item.n) continue;
                typename H::T* dst = static_cast<typename H::T*>(p.out) + (static_cast<size_t>(item.row0) + qrow) * p.D + item.head * ATT_HD + cq;
#pragma unroll
                for (int c = 0; c < 8; ++c)
                    *reinterpret_cast<uint32_t*>(dst + 8 * c) = H::pack(o[h][4 * c + 2 * r] * inv[r], o[h][4 * c + 2 * r + 1] * inv[r]);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ host
// Work list for `nimg` images packed back to back (image i: rows [row0[i], row0[i] + n[i])): one item per (image, head, pair of
// query tiles), ordered image-major / head / query pair so that the items sharing K/V are adjacent; `ranges` cuts the list into
// `ncta` contiguous pieces of (nearly) equal cost (cost of an item = kv tiles x query tiles it covers).
void attention_work_list(const int* row0, const int* n, int nimg, int heads, int ncta, std::vector<AttnItem>* items,
                         std::vector<int2>* ranges) {
    items->clear();
    std::vector<double> cost;
    for (int i = 0; i < nimg; ++i) {
        const int nq = (n[i] + 2 * ATT_BQ - 1) / (2 * ATT_BQ), nkv = (n[i] + ATT_BKV - 1) / ATT_BKV;
        for (int h = 0; h < heads; ++h)
            for (int q = 0; q < nq; ++q) {
                AttnItem it; it.row0 = row0[i]; it.n = n[i]; it.q0 = q * 2 * ATT_BQ; it.head = h;
                items->push_back(it);
                const int ng = (it.q0 + ATT_BQ < n[i]) ? 2 : 1;
                cost.push_back(static_cast<double>(nkv) * ng + 0.5);          // + per-item overhead (Q load, O store)
            }
    }
    const int total = static_cast<int>(items->size());
    if (ncta > total) ncta = total;
    ranges->assign(ncta > 0 ? ncta : 0, make_int2(0, 0));
    if (ncta <= 0) return;
    double sum = 0;
    for (double c : cost) sum += c;
    double acc = 0;
    int begin = 0, c = 0;
    for (int i = 0; i < total && c < ncta - 1; ++i) {
        acc += cost[i];
        const int items_left = total - (i + 1), ctas_left = ncta - (c + 1);
        if (acc >= sum * (c + 1) / ncta || items_left == ctas_left) {      // cut here (every CTA gets at least one item)
            (*ranges)[c++] = make_int2(begin, i + 1);
            begin = i + 1;
        }
    }
    (*ranges)[ncta - 1] = make_int2(begin, total);
}

int launch_attention(const CUtensorMap& mapQKV, void* out, const AttnItem* items_dev, const int2* ranges_dev, int ncta, int D, int heads,
                     bool bf16, cudaStream_t st) {
    if (D != heads * ATT_HD) return set_error("attention: head dim must be 64 (D=%d heads=%d)", D, heads);
    if (ncta <= 0) return 0;
    AttnParams p;
    p.out = out; p.items = items_dev; p.ranges = ranges_dev; p.D = D;
    p.scale_log2 = 0.125f * 1.4426950408889634f;
    auto kern = bf16 ? attention_kernel<true> : attention_kernel<false>;
    if (bf16) MG_SET_SMEM_ONCE(attention_kernel<true>, ATT_SMEM);
    else MG_SET_SMEM_ONCE(attention_kernel<false>, ATT_SMEM);
    CUDA_TRY(launch_pdl(kern, dim3(ncta), dim3(ATT_THREADS), ATT_SMEM, st, mapQKV, p));
    return 0;
}

}  // namespace mg
