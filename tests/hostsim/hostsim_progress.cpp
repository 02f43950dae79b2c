// TEST TOOL (not a product path): the host simulation of hostsim.cpp with the progress words of an astcenc_compress_image
// pass (astc_dev_lockstep.cuh, pass_cancelled). Every DevImage / BlockFeed the harness builds points at the two words below
// (ASTC_PASS_*_DEFAULT), so each compression runs with a cancel flag and a done counter:
//   hostsim_set_cancel(-1)  the flag stays down (default)
//   hostsim_set_cancel(0)   the flag is raised before the pass
//   hostsim_set_cancel(N)   the flag is raised at the N-th look at it (every pop and every ticket looks once)
//   hostsim_done()          the done counter of the last compression
// Built like hostsim.cpp, with one simulated lane or with -DASTC_HOSTSIM_LANES32=1.
#include <cstdint>
static uint32_t g_progress_flag = 0;
static uint32_t g_progress_done = 0;
#define ASTC_PASS_CANCEL_DEFAULT (&g_progress_flag)
#define ASTC_PASS_DONE_DEFAULT (&g_progress_done)
#include "hostsim.cpp"

static int g_cancel_at = -1;
static int g_cancel_looks = 0;
static void cancel_look() {
	if (g_cancel_at > 0 && ++g_cancel_looks >= g_cancel_at) {
		g_progress_flag = 1;
	}
}
extern "C" void hostsim_set_cancel(int at) { g_cancel_at = at; }
extern "C" unsigned int hostsim_done() { return g_progress_done; }

// hostsim_compress_volume with the words reset (and the flag raised first for hostsim_set_cancel(0))
extern "C" int hostsim_progress_volume(int profile, unsigned int bx, unsigned int by, unsigned int bz, float quality, unsigned int flags,
                                       const void* data, int data_type, unsigned int dim_x, unsigned int dim_y, unsigned int dim_z, const int* swz, uint8_t* out) {
	g_progress_flag = g_cancel_at == 0 ? 1u : 0u;
	g_progress_done = 0;
	g_cancel_looks = 0;
	g_hostsim_cancel_look = cancel_look;
	int rc = hostsim_compress_volume(profile, bx, by, bz, quality, flags, data, data_type, dim_x, dim_y, dim_z, swz, out);
	g_hostsim_cancel_look = nullptr;
	return rc;
}
