// TEST TOOL (not a product path): device block lists (astc_dev_gather.cuh) on the host simulation. Everything of
// hostsim_blocks.cpp, plus:
//   hostsim_gather_list  gather_block over the slots of one device block list (a one-entry block-list table), exactly as
//                        astc_gather_blocks_kernel runs it: the first min(*count, capacity) indices inside the image are
//                        gathered, every other slot (past the count, or out of range) is staged as zero texels and averages
// Built like hostsim_blocks.cpp, with one simulated lane or with -DASTC_HOSTSIM_LANES32=1.
#include "hostsim_blocks.cpp"

extern "C" void hostsim_gather_list(const void* src, int data_type, unsigned int dim_x, unsigned int dim_y, unsigned int dim_z, unsigned int bx,
                                    unsigned int by, unsigned int bz, const uint32_t* indices, uint32_t count, unsigned int capacity, const float* avg_src,
                                    void* dst, float* avg_dst) {
	GatherImage im{};
	im.data = src;
	im.dim_x = dim_x;
	im.dim_y = dim_y;
	im.dim_z = dim_z;
	im.blocks_x = (dim_x + bx - 1) / bx;
	im.blocks_y = (dim_y + by - 1) / by;
	GatherList l;
	l.indices = indices;
	l.count = &count;
	l.capacity = capacity;
	l.blocks = im.blocks_x * im.blocks_y * (bz > 1 ? (dim_z + bz - 1) / bz : dim_z);
	GatherArgs g;
	g.dst = dst;
	g.avg_src = avg_src;
	g.avg_dst = avg_dst;
	g.n = capacity;
	g.words = data_type == 0 ? 1 : data_type == 1 ? 2 : 4;
	g.bx = bx;
	g.by = by;
	g.bz = bz;
	g.images = &im;
	g.image_count = 1;
	g.lists = &l;
	run_lanes([&](int lane) {
		for (unsigned int i = 0; i < capacity; i++) {
			gather_block(g, i, lane, ASTC_WARP);
		}
	});
}
