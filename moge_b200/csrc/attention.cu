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
// list (cost-balanced, and dealt so that all CTAs run neighbouring items at once -> K/V come from L2; see attention_work_list).
// Warpgroup 0 streams Q and the K/V ring by TMA; consumer warpgroup g (1 + g) owns query tile g of the item and runs it as two
// 64-row halves, each with its own O accumulator and running max / sum.
//
// BURSTS.  A consumer issues its MMAs in bursts, one commit group and one wait each, and between two bursts runs the softmax of
// one half.  With K/V tiles j = 0 .. nkv-1 and halves h0, h1, an item is
//     {S h0(0)} sm h0 {PV h0(0), S h1(0)} sm h1 {PV h1(0), S h0(1)} sm h0 ... {PV h0(last), S h1(last)} sm h1 {PV h1(last)}
// then the normalise and store: 2 nkv + 1 bursts.  Every MMA keeps its operands and k-order and every softmax its arithmetic,
// so the results are bit for bit those of running each half's S, softmax and P V one after another.
// DEAD TILES.  When item.q0 + 128 >= item.n (the last item of an image whose second query tile lies past the image), consumer 1
// has no rows: the Q warp loads one Q tile, and consumer 1 issues no MMA and stores nothing.
// PRODUCERS.  Warp 0 loads the Q tiles, warp 1 streams the K/V ring.  The ring does not wait for the next item's Q, so the next
// item's first K/V tiles load under the end of the current one; Q loads once the current item's last S has completed.
//
// Barrier protocol (every wait is an mbar_wait, whose watchdog turns a protocol error into a launch failure):
//   barrier      count  arrivals                                                     waited by
//   q_full       1+tx   Q warp (expect_tx of the Q tiles it loads)                   every consumer warp, at the item's start
//   q_empty      8      every consumer warp, after {PV h0(last), S h1(last)}         Q warp, before the next item's Q
//   k_full[s]    1+tx   K/V warp                                                     the burst holding S h0(j)
//   k_empty[s]   8      every consumer warp, after {PV h0(j), S h1(j)} completed     K/V warp, before it reloads slot s
//   v_full[s]    1+tx   K/V warp                                                     the burst {PV h0(j), S h1(j)}
//   v_empty[s]   8      every consumer warp, after {PV h1(j), ...} completed         K/V warp, before it reloads slot s
// A consumer warp that owns a dead tile waits q_full, then k_full / v_full of every tile, and arrives on q_empty, k_empty and
// v_empty after each: waiting first keeps its arrival in the phase that the tile's readers complete (a slot or the Q buffer is
// refilled only after that phase).
// Why every wait is satisfied.  The K/V warp refills slot s with tile j after the releases of tile j-5, which come with the
// bursts {PV h0(j-5), S h1(j-5)} and {PV h1(j-5), S h0(j-4)}; both complete before the first burst that reads tile j,
// {PV h1(j-1), S h0(j)}, is issued.  It loads K_0 V_0 K_1 V_1 ... in order (across items too), so each of its waits needs only
// releases from earlier bursts.  The Q warp loads item i+1's Q after q_empty of item i, which both consumers arrive on before
// their last burst of item i, and no consumer waits on anything of item i+1 before it has finished item i.  So no wait depends
// on a later event, and every barrier is at most one phase ahead of its slowest waiter, so a parity wait cannot miss a phase.
#include "common.cuh"
#include "host_api.h"
#include <functional>
#include <queue>
#include <utility>
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

// S = Q K^T of one 64-row half, accumulated into sv (the caller zeroes it: scale-d = 1, as the sums always started from +0)
template <bool BF16>
__device__ __forceinline__ void att_issue_s(float (&sv)[64], uint64_t qd, uint64_t kd) {
#pragma unroll
    for (int k = 0; k < ATT_HD / 16; ++k) Wgmma<ATT_BKV, BF16>::ss(sv, qd + 2 * k, kd + 2 * k, 1u);
}
// O += P V of one 64-row half, P from registers
template <bool BF16>
__device__ __forceinline__ void att_issue_pv(float (&o)[32], const uint32_t (&pa)[32], uint32_t vaddr) {
#pragma unroll
    for (int kk = 0; kk < ATT_BKV / 16; ++kk) {
        // B: V tile [kv][hd], MN-major, 16 kv rows (= 2 groups of 8 x 128 B) per K-step
        const uint64_t vd = make_sdesc_sw128(vaddr + kk * 16 * 128, /*lbo=*/ATT_TILE_BYTES, /*sbo=*/1024);
        wgmma_rs_n64_tb<BF16>(o, pa + 4 * kk, vd, 1u);
    }
}
__device__ __forceinline__ void att_zero(float (&sv)[64]) {
#pragma unroll
    for (int i = 0; i < 64; ++i) sv[i] = 0.f;
}
// Online softmax of one 64-row half: masks the padding columns of the last K/V tile, updates the running max m and sum l,
// rescales o and packs P = 2^(S sc - m sc) to 16 bit in the A-operand fragment order of the P V MMA (k-step kk: columns 16 kk ..)
template <bool BF16>
__device__ __forceinline__ void att_softmax(float (&sv)[64], uint32_t (&pa)[32], float (&o)[32], float (&m)[2], float (&l)[2],
                                            int kv_left, int cq, float sc) {
    using H = H16<BF16>;
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
        const float m_new = fmaxf(m[r], mx[r]);
        alpha[r] = ex2_approx((m[r] - m_new) * sc);        // 0 on the first tile (m = -inf)
        m[r] = m_new;
        mb[r] = m_new * sc;
        l[r] *= alpha[r];
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] *= alpha[(i >> 1) & 1];
#pragma unroll
    for (int i = 0; i < 64; i += 2) {
        const int r = (i >> 1) & 1;
        const float e0 = ex2_approx(fmaf(sv[i], sc, -mb[r])), e1 = ex2_approx(fmaf(sv[i + 1], sc, -mb[r]));
        l[r] += e0 + e1;
        pa[i >> 1] = H::pack(e0, e1);
    }
}

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
        // ============================================ TMA producers (converged warps, one elected lane issues): warp 0 loads the
        // Q tiles, warp 1 streams the K/V ring.  The ring does not wait for the next item's Q: its first tiles load under the end
        // of the current item.
        regs_dec<40>();
        if (warp == 0) {
            for (int it = rng.x; it < rng.y; ++it) {
                const AttnItem item = p.items[it];
                const int li = it - rng.x;
                if (li > 0) mbar_wait(q_empty, (li - 1) & 1);
                if (elect_one()) {
                    // the second query tile only when it holds rows of the image (no consumer reads it otherwise)
                    const bool two = item.q0 + ATT_BQ < item.n;
                    mbar_arrive_expect_tx(q_full, (two ? 2 : 1) * ATT_TILE_BYTES);
                    tma_load_2d(sQ, &mapQKV, q_full, item.head * ATT_HD, item.row0 + item.q0);
                    if (two) tma_load_2d(sQ + ATT_TILE_BYTES, &mapQKV, q_full, item.head * ATT_HD, item.row0 + item.q0 + ATT_BQ);
                }
                __syncwarp();
            }
        } else if (warp == 1) {
            int s = 0; uint32_t ph = 0;
            for (int it = rng.x; it < rng.y; ++it) {
                const AttnItem item = p.items[it];
                const int nkv = (item.n + ATT_BKV - 1) / ATT_BKV;
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
        }
        return;
    }
    // ============================================================== consumers: bursts of S = Q K^T and O += P V, softmax between
    regs_inc<232>();
    const int g = (warp - 4) >> 2;          // query tile of the item
    const int wl = warp & 3;
    const float sc = p.scale_log2;
    // accumulator fragment: this thread's rows r0 and r0 + 8 of a 64-row half; columns 8 (i / 4) + 2 (lane % 4) + i % 2
    const int r0 = 16 * wl + (lane >> 2);
    const int cq = 2 * (lane & 3);
    auto arrive = [&](uint64_t* bar) {      // one arrival per warp
        __syncwarp();
        if (lane == 0) mbar_arrive(bar);
    };
    int s = 0; uint32_t ph = 0;
    for (int it = rng.x; it < rng.y; ++it) {
        const AttnItem item = p.items[it];
        const int li = it - rng.x;
        const int nkv = (item.n + ATT_BKV - 1) / ATT_BKV;
        mbar_wait(q_full, li & 1);
        if (g == 1 && item.q0 + ATT_BQ >= item.n) {
            // dead tile: no MMA, no store; keep every arrival the protocol counts
            for (int j = 0; j < nkv; ++j) {
                mbar_wait(&k_full[s], ph);
                arrive(&k_empty[s]);
                mbar_wait(&v_full[s], ph);
                arrive(&v_empty[s]);
                if (++s == ST) { s = 0; ph ^= 1; }
            }
            arrive(q_empty);
            continue;
        }
        float o0[32], o1[32];
        float m0[2] = {-INFINITY, -INFINITY}, m1[2] = {-INFINITY, -INFINITY};
        float l0[2] = {0.f, 0.f}, l1[2] = {0.f, 0.f};
#pragma unroll
        for (int i = 0; i < 32; ++i) o0[i] = o1[i] = 0.f;
        const uint64_t qd0 = make_sdesc_sw128(smem_u32(sQ + g * ATT_TILE_BYTES));
        const uint64_t qd1 = make_sdesc_sw128(smem_u32(sQ + g * ATT_TILE_BYTES + 64 * 128));
        float sv[64];
        uint32_t pa[32];
        // {S h0(0)}
        mbar_wait(&k_full[s], ph);
        att_zero(sv);
        wgmma_fence();
        att_issue_s<BF16>(sv, qd0, make_sdesc_sw128(smem_u32(sK + s * ATT_TILE_BYTES)));
        wgmma_commit();
        wgmma_wait<0>();
        reg_fence(sv);
        for (int j = 0;; ++j) {
            const int kv_left = item.n - j * ATT_BKV;
            const uint32_t vaddr = smem_u32(sV + s * ATT_TILE_BYTES);
            att_softmax<BF16>(sv, pa, o0, m0, l0, kv_left, cq, sc);
            // {PV h0(j), S h1(j)}: the tile's second S -> its K slot is free
            mbar_wait(&v_full[s], ph);
            att_zero(sv);
            wgmma_fence();
            att_issue_pv<BF16>(o0, pa, vaddr);
            att_issue_s<BF16>(sv, qd1, make_sdesc_sw128(smem_u32(sK + s * ATT_TILE_BYTES)));
            wgmma_commit();
            wgmma_wait<0>();
            reg_fence(sv);
            reg_fence(o0);
            arrive(&k_empty[s]);
            if (j + 1 == nkv) arrive(q_empty);      // the item's last S has completed: the next item's Q may load
            att_softmax<BF16>(sv, pa, o1, m1, l1, kv_left, cq, sc);
            if (j + 1 == nkv) break;
            // {PV h1(j), S h0(j+1)}: the tile's second P V -> its V slot is free
            const int sn = s + 1 == ST ? 0 : s + 1;
            const uint32_t phn = s + 1 == ST ? ph ^ 1 : ph;
            mbar_wait(&k_full[sn], phn);
            att_zero(sv);
            wgmma_fence();
            att_issue_pv<BF16>(o1, pa, vaddr);
            att_issue_s<BF16>(sv, qd0, make_sdesc_sw128(smem_u32(sK + sn * ATT_TILE_BYTES)));
            wgmma_commit();
            wgmma_wait<0>();
            reg_fence(sv);
            reg_fence(o1);
            arrive(&v_empty[s]);
            s = sn; ph = phn;
        }
        // {PV h1(last)}
        wgmma_fence();
        att_issue_pv<BF16>(o1, pa, smem_u32(sV + s * ATT_TILE_BYTES));
        wgmma_commit();
        wgmma_wait<0>();
        reg_fence(o1);
        arrive(&v_empty[s]);
        if (++s == ST) { s = 0; ph ^= 1; }
        // normalise + store
        const int live_rows = item.n - item.q0 - g * ATT_BQ;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float (&o)[32] = h == 0 ? o0 : o1;
            float (&l)[2] = h == 0 ? l0 : l1;
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
                l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
            }
            const float inv[2] = {1.0f / l[0], 1.0f / l[1]};
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const int q = h * 64 + r0 + 8 * r;
                if (q >= live_rows) continue;
                const int qrow = item.q0 + g * ATT_BQ + q;
                typename H::T* dst = static_cast<typename H::T*>(p.out) + (static_cast<size_t>(item.row0) + qrow) * p.D + item.head * ATT_HD + cq;
#pragma unroll
                for (int c = 0; c < 8; ++c)
                    *reinterpret_cast<uint32_t*>(dst + 8 * c) = H::pack(o[4 * c + 2 * r] * inv[r], o[4 * c + 2 * r + 1] * inv[r]);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ host
// Work list for `nimg` images packed back to back (image i: n[i] rows): one item per (image, head, pair of
// query tiles).  The items are dealt out in image-major / head / query-pair order, each to the CTA with the least modelled cost
// so far (cost of an item = kv tiles x query tiles it covers; lowest CTA index on ties), and the list is returned CTA by CTA, so
// that `ranges` gives each CTA a contiguous piece.  Since every CTA walks its items in that order and the costs track the time,
// the CTAs run neighbouring items of the dealing order at any moment: the K/V of the few (image, head)s in flight (132 SMs over
// the 6 items of a 1370-token image: about 22, 8 MB) stay in L2 for all their readers.  (Handing each CTA a run of consecutive
// items of one (image, head) instead kept 132 of them in flight, 46 MB of K/V, and the kernel re-read K/V at about 2.2 TB/s.)
// List scheduling keeps every CTA within one item's cost of the mean.
void attention_work_list(const int* n, int nimg, int heads, int ncta, std::vector<AttnItem>* items, std::vector<int2>* ranges) {
    std::vector<AttnItem> order;
    std::vector<double> cost;
    int row0 = 0;
    for (int i = 0; i < nimg; ++i) {
        const int nq = (n[i] + 2 * ATT_BQ - 1) / (2 * ATT_BQ), nkv = (n[i] + ATT_BKV - 1) / ATT_BKV;
        for (int h = 0; h < heads; ++h)
            for (int q = 0; q < nq; ++q) {
                AttnItem it; it.row0 = row0; it.n = n[i]; it.q0 = q * 2 * ATT_BQ; it.head = h;
                order.push_back(it);
                const int ng = (it.q0 + ATT_BQ < n[i]) ? 2 : 1;
                cost.push_back(static_cast<double>(nkv) * ng + 0.5);          // + per-item overhead (Q load, O store)
            }
        row0 += n[i];
    }
    const int total = static_cast<int>(order.size());
    if (ncta > total) ncta = total;
    items->clear();
    ranges->assign(ncta > 0 ? ncta : 0, make_int2(0, 0));
    if (ncta <= 0) return;
    // min-heap of (modelled cost so far, CTA): the first ncta items go to CTAs 0 .. ncta-1, so every CTA gets at least one
    std::priority_queue<std::pair<double, int>, std::vector<std::pair<double, int>>, std::greater<std::pair<double, int>>> load;
    for (int c = 0; c < ncta; ++c) load.push({0.0, c});
    std::vector<std::vector<int>> per_cta(ncta);
    for (int i = 0; i < total; ++i) {
        const std::pair<double, int> least = load.top();
        load.pop();
        per_cta[least.second].push_back(i);
        load.push({least.first + cost[i], least.second});
    }
    for (int c = 0; c < ncta; ++c) {
        const int begin = static_cast<int>(items->size());
        for (int i : per_cta[c]) items->push_back(order[i]);
        (*ranges)[c] = make_int2(begin, static_cast<int>(items->size()));
    }
}

int upload_attention_work(const std::vector<int>& n, int heads, int ncta, const std::function<int(void**, size_t)>& alloc, cudaStream_t st,
                          AttnWork* w) {
    attention_work_list(n.data(), static_cast<int>(n.size()), heads, ncta, &w->items, &w->ranges);
    MG_TRY(alloc(reinterpret_cast<void**>(&w->items_dev), w->items.size() * sizeof(AttnItem) + 16));
    MG_TRY(alloc(reinterpret_cast<void**>(&w->ranges_dev), w->ranges.size() * sizeof(int2) + 16));
    CUDA_TRY(cudaMemcpyAsync(w->items_dev, w->items.data(), w->items.size() * sizeof(AttnItem), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(w->ranges_dev, w->ranges.data(), w->ranges.size() * sizeof(int2), cudaMemcpyHostToDevice, st));
    return 0;
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
