// kernel_deal.cuh -- the static-deal driver shared by k_long_s, k_mid, k_short and k_short_g (device code; included by
// kernel_long.cuh after the mbarrier / TMA primitives it builds on).
//
// A launch of n items -- a run, or a group of runs transformed in lockstep -- deals them to its W warps statically: item
// i goes to warp i mod W (W from static_deal_grid).  Every warp then knows its whole future, so the latencies of an item
// (descriptor, state rows, first tiles) overlap with the arithmetic of the items before it:
//   * descriptors: an item's descriptor, Quads 16-byte quads, is copied by cp.async, one quad per lane, into a ring of
//     Slots shared-memory slots, Fetch items ahead of the producer;
//   * producer: a warp-uniform cursor (item, unit, descriptor slot, stage) walks the warp's units -- packets, or octets
//     of packets -- in processing order and issues each unit's TMA copies into the next of Ring stages, counted on that
//     stage's mbarrier.  It stays Ring stages ahead of the consumer across any number of item boundaries.  The kernel
//     says how many units an item has and how one unit is issued; the driver owns the order, the wrap and the advance;
//   * consumer: waits on its stage with the stage's phase bit and hands the stage back by calling the producer (a
//     stage doubles as the transpose scratch, so only the consumer knows when it is free);
//   * state rows (k_long_s, k_mid): one more tile, on mbarrier Ring, takes the state rows of the next item that reads
//     some.  They are requested as soon as the tile is free and that item's descriptor has landed.  The kernel says
//     which items need rows and how they are issued.
// Slots >= Fetch + Ring + 1: a fetch never overwrites the descriptor of an item the consumer or the producer is on.
#pragma once

namespace lwb {

// Grid of a static deal of n items over CTAs of `warps` warps, at most one CTA per SM.  The host balances the deal for
// W = grid * warps (balance_static_deal) and the kernel deals with gridDim.x * warps: both come from here.
inline uint32_t static_deal_grid(size_t n, int warps, int sm_count)
{
    const size_t want = (n + warps - 1) / warps;
    return (uint32_t)(want < (size_t)sm_count ? want : (size_t)sm_count);
}

__device__ __forceinline__ void cp_async16(uint32_t dst, const void *src)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

template <int N>
__device__ __forceinline__ uint32_t ring_next(uint32_t x) { return x + 1 == (uint32_t)N ? 0 : x + 1; }

template <int Quads, int Slots, int Fetch, int Ring, uint32_t StageBytes>
struct StaticDeal {
    static_assert(Slots >= Fetch + Ring + 1, "a descriptor fetch would overwrite a slot still in use");
    static_assert(Ring < 30, "phase bit 30 belongs to the state tile");
    const uint4 *src;
    uint32_t n, W, desc_s, ring_s, bars_s;
    int lane;
    uint32_t f_idx, f_slot = 0;                                            // next descriptor to fetch
    uint32_t p_idx, p_unit = 0, p_slot = 0, p_stage = 0;                  // producer
    uint32_t c_slot = 0, c_stage = 0, phase_bits = 0;                      // consumer
    uint32_t st_idx = ~0u;                         // the item whose state rows are in the tile or on their way (~0: free)

    // gw < n: the warp's first item.  desc_s, ring_s, bars_s: the warp's descriptor slots, stages and mbarriers.
    __device__ __forceinline__ StaticDeal(const void *descs, uint32_t n_, uint32_t W_, uint32_t gw, uint32_t desc_s_,
                                          uint32_t ring_s_, uint32_t bars_s_, int lane_)
        : src(reinterpret_cast<const uint4 *>(descs)), n(n_), W(W_), desc_s(desc_s_), ring_s(ring_s_), bars_s(bars_s_),
          lane(lane_), f_idx(gw), p_idx(gw)
    {
    }

    // cp.async groups are per thread: every lane commits and waits, whether it copied a quad or not
    __device__ __forceinline__ void fetch()
    {
        if ((uint32_t)lane < (uint32_t)Quads && f_idx < n)
            cp_async16(desc_s + f_slot * (16u * Quads) + 16u * (uint32_t)lane, src + (size_t)Quads * f_idx + lane);
        cp_async_commit();
        f_idx += W;
        f_slot = ring_next<Slots>(f_slot);
    }

    // Whole warp.  units(slot): units of the item whose descriptor is in `slot`.  issue(slot, unit, bar, dst): arm the
    // mbarrier at `bar` and start the unit's copies into the stage at `dst`.
    template <class Units, class Issue>
    __device__ __forceinline__ void start(Units units, Issue issue)
    {
#pragma unroll
        for (int i = 0; i <= Fetch; i++) fetch();
        cp_async_wait<Fetch>();
        __syncwarp();
        for (int i = 0; i < Ring; i++) produce(units, issue);
    }
    // the next unit, into the stage the consumer has just freed (nothing once the warp's items are exhausted)
    template <class Units, class Issue>
    __device__ __forceinline__ void produce(Units units, Issue issue)
    {
        if (p_idx >= n) return;
        issue(p_slot, p_unit, bars_s + 8u * p_stage, ring_s + p_stage * StageBytes);
        p_stage = ring_next<Ring>(p_stage);
        if (++p_unit >= units(p_slot)) {
            p_idx += W;
            p_unit = 0;
            p_slot = ring_next<Slots>(p_slot);
            fetch();                      // item p_idx + Fetch W
            cp_async_wait<Fetch>();       // item p_idx's descriptor has landed
            __syncwarp();
        }
    }

    // consumer: the descriptor slot of the next item; the stage of the next unit once its copies have landed
    __device__ __forceinline__ uint32_t take_slot()
    {
        const uint32_t s = c_slot;
        c_slot = ring_next<Slots>(c_slot);
        return s;
    }
    __device__ __forceinline__ uint32_t wait_stage()
    {
        mbar_wait(bars_s + 8u * c_stage, (phase_bits >> c_stage) & 1u);
        phase_bits ^= 1u << c_stage;
        return c_stage;
    }
    __device__ __forceinline__ void next_stage() { c_stage = ring_next<Ring>(c_stage); }

    // State rows, whole warp.  needs(slot): the item in `slot` reads rows.  issue(slot, bar): arm `bar` and start them.
    // request_state: the first item in [from, p_idx] that needs rows -- the descriptors between the consumer and the
    // producer have landed and stay until the consumer has passed them.
    template <class Needs, class IssueState>
    __device__ __forceinline__ void request_state(uint32_t from, uint32_t sl, Needs needs, IssueState issue)
    {
        while (from < n && from <= p_idx) {
            if (needs(sl)) {
                issue(sl, bars_s + 8u * Ring);
                st_idx = from;
                return;
            }
            from += W;
            sl = ring_next<Slots>(sl);
        }
    }
    // the descriptor slot of the item being consumed (take_slot has moved past it)
    __device__ __forceinline__ uint32_t consumer_slot() const { return c_slot == 0 ? Slots - 1 : c_slot - 1; }
    // item c, the one being consumed, starts: look ahead if the tile is free
    template <class Needs, class IssueState>
    __device__ __forceinline__ void begin_state(uint32_t c, Needs needs, IssueState issue)
    {
        if (st_idx == ~0u) request_state(c, consumer_slot(), needs, issue);
    }
    // item c reads its rows now: issue them if its descriptor had not landed when the tile came free, and wait
    template <class IssueState>
    __device__ __forceinline__ void wait_state(uint32_t c, IssueState issue)
    {
        if (st_idx != c) {
            issue(consumer_slot(), bars_s + 8u * Ring);
            st_idx = c;
        }
        mbar_wait(bars_s + 8u * Ring, (phase_bits >> 30) & 1u);
        phase_bits ^= 1u << 30;
    }
    // item c has consumed the tile: on to the next item that needs it
    template <class Needs, class IssueState>
    __device__ __forceinline__ void release_state(uint32_t c, Needs needs, IssueState issue)
    {
        st_idx = ~0u;
        request_state(c + W, c_slot, needs, issue);
    }
};

}  // namespace lwb
