// TEST TOOL (not a product path): image tables (astc_dev_gather.cuh) on the host simulation of hostsim.cpp. Everything of
// hostsim_blocks.cpp, plus:
//   hostsim_gather_images   gather_block over staging blocks [base, base + n) of a table of images, exactly as
//                           astc_gather_blocks_kernel runs it (one simulated lane)
//   hostsim_scatter_images  scatter_target for the same staging blocks: each staged block to its image's payload
// The table is built as astcenc_b200_compress_device_images builds it: first[] is the exclusive prefix sum of the images' block
// counts, and each image's averages follow those of the images before it (dim_x * dim_y floats each).
#include "hostsim_blocks.cpp"

static std::vector<GatherImage> image_table(const void* const* data, const unsigned int* dims, unsigned int image_count, unsigned int bx, unsigned int by,
                                            unsigned int bz, uint8_t* const* payloads) {
	std::vector<GatherImage> table(image_count);
	size_t first = 0, avg_offset = 0;
	for (unsigned int j = 0; j < image_count; j++) {
		GatherImage& e = table[j];
		e.data = data[j];
		e.payload = payloads != nullptr ? payloads[j] : nullptr;
		e.dim_x = dims[3 * j];
		e.dim_y = dims[3 * j + 1];
		e.dim_z = dims[3 * j + 2];
		e.blocks_x = (e.dim_x + bx - 1) / bx;
		e.blocks_y = (e.dim_y + by - 1) / by;
		e.first = first;
		e.avg_offset = avg_offset;
		first += (size_t)e.blocks_x * e.blocks_y * ((e.dim_z + bz - 1) / bz);
		avg_offset += (size_t)e.dim_x * e.dim_y;
	}
	return table;
}

static GatherArgs table_args(const std::vector<GatherImage>& table, int data_type, unsigned int bx, unsigned int by, unsigned int bz, size_t base,
                             unsigned int n) {
	GatherArgs g;
	g.src = nullptr;
	g.dst = nullptr;
	g.avg_src = nullptr;
	g.avg_dst = nullptr;
	g.indices = nullptr;
	g.n = n;
	g.words = data_type == 0 ? 1 : data_type == 1 ? 2 : 4;
	g.dim_x = g.dim_y = g.dim_z = 0;
	g.blocks_x = g.blocks_y = 0;
	g.bx = bx;
	g.by = by;
	g.bz = bz;
	g.images = table.data();
	g.image_count = (unsigned int)table.size();
	g.base = base;
	return g;
}

extern "C" void hostsim_gather_images(const void* const* data, const unsigned int* dims, unsigned int image_count, int data_type, unsigned int bx,
                                      unsigned int by, unsigned int bz, size_t base, unsigned int n, const float* avg_src, void* dst, float* avg_dst) {
	std::vector<GatherImage> table = image_table(data, dims, image_count, bx, by, bz, nullptr);
	GatherArgs g = table_args(table, data_type, bx, by, bz, base, n);
	g.dst = dst;
	g.avg_src = avg_src;
	g.avg_dst = avg_dst;
	for (unsigned int i = 0; i < n; i++) {
		gather_block(g, i, 0, 1);
	}
}

extern "C" void hostsim_scatter_images(const unsigned int* dims, unsigned int image_count, unsigned int bx, unsigned int by, unsigned int bz, size_t base,
                                       unsigned int n, const uint8_t* staged, uint8_t* const* payloads) {
	std::vector<const void*> none(image_count, nullptr);
	std::vector<GatherImage> table = image_table(none.data(), dims, image_count, bx, by, bz, payloads);
	GatherArgs g = table_args(table, 0, bx, by, bz, base, n);
	for (unsigned int i = 0; i < n; i++) {
		memcpy(scatter_target(g, i, nullptr), staged + (size_t)i * 16, 16);
	}
}
