// TEST TOOL (not a product path): packed block-list tables (astc_dev_pack.cuh, the PACKED staged_block of astc_dev_gather.cuh)
// on the host simulation. Everything of hostsim_refine.cpp, plus:
//   hostsim_pack_lists            pack_lists over a table, as astc_pack_lists_kernel runs it (one lane or 32)
//   hostsim_pack_slots            the packed resolution of staging slots [base, base + n) after the packing
//   hostsim_unpacked_slots        the unpacked resolution of the same lists (it reads slots past the count: the stray-read check's
//                                 positive control)
//   hostsim_refine_decide_packed  refine_decide_block<M, true> over staging blocks [base, base + n) of a packed refine call
//   hostsim_refine_commit_packed  refine_commit_block<true> over the same staging blocks
// Every ASTC_LDG of the device source is checked here: a read of list memory the rule forbids (an index at or beyond
// min(*count, capacity) of its list, or the count of a list of capacity 0) is counted, and each call returns the count.
// Tables are built as the library builds them (plan_blocks): entries of capacity 0 are left out.
#include <atomic>
#include <cstdint>
#include <vector>

struct ForbiddenRange {
	uintptr_t lo, hi;
};
static std::vector<ForbiddenRange> g_forbidden;
static std::atomic<unsigned int> g_stray_reads{0};

template <typename T> static inline T hostsim_checked_ldg(const T* p) {
	const uintptr_t a = reinterpret_cast<uintptr_t>(p);
	for (const ForbiddenRange& r : g_forbidden) {
		if (a + sizeof(T) > r.lo && a < r.hi) {
			g_stray_reads++;
		}
	}
	return *p;
}
#define ASTC_LDG(p) hostsim_checked_ldg(p)

#include "hostsim_refine.cpp"
#include "../../astc-encoder_b200/csrc/astc_dev_pack.cuh"

// Words read past a list's listed slots count as stray up to this far beyond its capacity (the tests pad their lists by as much).
#define PACK_GUARD_WORDS 64

// Forbid the list memory of count entries that the rule never reads, and clear the stray count.
static void forbid_lists(const uint32_t* const* indices, const uint32_t* counts, const unsigned int* capacities, unsigned int count) {
	g_forbidden.clear();
	g_stray_reads = 0;
	for (unsigned int j = 0; j < count; j++) {
		if (capacities[j] == 0) {
			g_forbidden.push_back({reinterpret_cast<uintptr_t>(counts + j), reinterpret_cast<uintptr_t>(counts + j + 1)});
			continue;
		}
		const uint32_t v = counts[j] < capacities[j] ? counts[j] : capacities[j];
		g_forbidden.push_back({reinterpret_cast<uintptr_t>(indices[j] + v), reinterpret_cast<uintptr_t>(indices[j] + capacities[j] + PACK_GUARD_WORDS)});
	}
}

static unsigned int stray_reads() {
	g_forbidden.clear();
	return g_stray_reads.load();
}

// The packing of a staging table (entries of capacity > 0 only) into its firsts and the sentinel after it.
static void pack_table(std::vector<GatherImage>& table, const std::vector<GatherList>& lists, uint32_t budget, uint32_t* overflow) {
	const unsigned int count = (unsigned int)lists.size();
	table.resize(count + 1);      // (the sentinel)
	run_lanes([&](int lane) { pack_lists(table.data(), lists.data(), count, budget, overflow, lane, ASTC_WARP); });
}

// A packed table of `count` entries (list j: indices[j], counts + j, capacities[j], blocks[j]), packed under `budget`. order[k]:
// the caller's entry of table entry k.
struct SimPacked {
	std::vector<GatherImage> table;
	std::vector<GatherList> lists;
	std::vector<unsigned int> order;
	SimPacked(const uint32_t* const* indices, const uint32_t* counts, const unsigned int* capacities, const unsigned int* blocks, unsigned int count,
	          uint32_t budget, uint32_t* overflow) {
		for (unsigned int j = 0; j < count; j++) {
			if (capacities[j] != 0) {
				lists.push_back({indices[j], counts + j, capacities[j], blocks[j]});
				order.push_back(j);
			}
		}
		pack_table(table, lists, budget, overflow);
	}
};

// The packing of `count` lists (counts[j], capacities[j]; indices are never read): firsts[j] the packed first of entry j
// (0xFFFFFFFFFFFFFFFF for an entry of capacity 0, which has none), *total the sentinel's first, *overflow (when not null).
// Returns the stray reads.
extern "C" unsigned int hostsim_pack_lists(const uint32_t* counts, const unsigned int* capacities, unsigned int count, uint32_t budget, uint64_t* firsts,
                                           uint64_t* total, uint32_t* overflow) {
	std::vector<const uint32_t*> none(count, nullptr);
	std::vector<unsigned int> blocks(count, 0);
	forbid_lists(none.data(), counts, capacities, count);
	SimPacked p(none.data(), counts, capacities, blocks.data(), count, budget, overflow);
	for (unsigned int j = 0; j < count; j++) {
		firsts[j] = ~0ull;
	}
	for (size_t k = 0; k < p.order.size(); k++) {
		firsts[p.order[k]] = p.table[k].first;
	}
	*total = p.order.empty() ? 0 : p.table[p.order.size()].first;
	return stray_reads();
}

// The packed resolution of staging slots base + i, i < n: entries[i] the caller's entry and blocks_out[i] the block, or
// 0xFFFFFFFF in both for an invalid slot. The lists: indices[j] (capacities[j] words, then PACK_GUARD_WORDS), counts[j],
// capacities[j] and the image's block count blocks[j]. Returns the stray reads.
extern "C" unsigned int hostsim_pack_slots(const uint32_t* const* indices, const uint32_t* counts, const unsigned int* capacities, const unsigned int* blocks,
                                           unsigned int count, uint32_t budget, size_t base, unsigned int n, uint32_t* entries, uint32_t* blocks_out) {
	forbid_lists(indices, counts, capacities, count);
	SimPacked p(indices, counts, capacities, blocks, count, budget, nullptr);
	GatherArgs g{};
	g.images = p.table.data();
	g.image_count = (unsigned int)p.lists.size();
	g.lists = p.lists.data();
	g.base = base;
	g.n = n;
	run_lanes([&](int lane) {
		for (unsigned int i = 0; i < n; i++) {
			unsigned int j;
			const uint32_t index = staged_block<true>(g, i, j);
			if (lane == 0) {
				entries[i] = index == GATHER_INVALID ? GATHER_INVALID : p.order[j];
				blocks_out[i] = index;
			}
		}
	});
	return stray_reads();
}

// The unpacked resolution (staged_block<false>) of staging slots base + i, i < n, of the same lists, as hostsim_pack_slots
// returns it. Returns the stray reads.
extern "C" unsigned int hostsim_unpacked_slots(const uint32_t* const* indices, const uint32_t* counts, const unsigned int* capacities,
                                               const unsigned int* blocks, unsigned int count, size_t base, unsigned int n, uint32_t* entries,
                                               uint32_t* blocks_out) {
	forbid_lists(indices, counts, capacities, count);
	std::vector<GatherImage> table;
	std::vector<GatherList> lists;
	std::vector<unsigned int> order;
	size_t first = 0;
	for (unsigned int j = 0; j < count; j++) {
		if (capacities[j] != 0) {
			GatherImage e{};
			e.first = first;
			table.push_back(e);
			lists.push_back({indices[j], counts + j, capacities[j], blocks[j]});
			order.push_back(j);
			first += capacities[j];
		}
	}
	GatherArgs g{};
	g.images = table.data();
	g.image_count = (unsigned int)lists.size();
	g.lists = lists.data();
	g.base = base;
	g.n = n;
	for (unsigned int i = 0; i < n; i++) {
		unsigned int j;
		const uint32_t index = staged_block(g, i, j);
		entries[i] = index == GATHER_INVALID ? GATHER_INVALID : order[j];
		blocks_out[i] = index;
	}
	return stray_reads();
}

// A packed refine call's chunk: SimRefine's table, packed under `budget`.
struct SimRefinePacked : SimRefine {
	template <typename... A> SimRefinePacked(uint32_t budget, A... a) : SimRefine(a...) {
		pack_table(table, lists, budget, nullptr);
		g.images = table.data();
	}
};

// The decisions of packed staging blocks [base, base + n) for maps of `block_metric`. Returns the stray reads.
extern "C" unsigned int hostsim_refine_decide_packed(SIM_REFINE_PARAMS, int block_metric, uint32_t budget) {
	forbid_lists(indices, counts, capacities, count);
	SimRefinePacked c(budget, SIM_REFINE_ARGS);
	with_metric(block_metric, [&](auto m) {
		run_lanes([&](int lane) {
			for (unsigned int i = 0; i < n; i++) {
				refine_decide_block<decltype(m)::value, true>(c.g, c.r, i, lane, ASTC_WARP);
			}
		});
	});
	return stray_reads();
}

// The commits of the same staging blocks; staged: their candidates, 16 bytes each. Returns the stray reads.
extern "C" unsigned int hostsim_refine_commit_packed(SIM_REFINE_PARAMS, const uint8_t* staged, uint32_t budget) {
	forbid_lists(indices, counts, capacities, count);
	SimRefinePacked c(budget, SIM_REFINE_ARGS);
	run_lanes([&](int lane) {
		for (unsigned int i = 0; i < n; i++) {
			refine_commit_block<true>(c.g, c.r, staged, i, lane, ASTC_WARP);
		}
	});
	return stray_reads();
}
