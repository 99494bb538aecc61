// The point-set handle's side of b200mvs_pset_add_reconstruction.  b200mvs.cu runs the reconstruction and hands every
// finished depth map, still on the device, to the handle of depthmap.cu together with the view's pyramid level and camera;
// each view's points are staged behind the handle's set and committed in the caller's view order when the whole call
// succeeded.
#pragma once
#include "../../include/b200mvs.h"

#include <cuda_runtime.h>

#include <cstdint>
#include <vector>

namespace b200mvs_pset_dev {

// The point set of a handle: lists of 4-byte items, PER[k] of them per entry (PIX: the (x, y) of each point for the
// correspondence).  They live in device memory for a handle made by b200mvs_pset_create_on_device and in host memory
// otherwise.  List k holds n[k] committed entries followed by staged[k] entries that a view appended and that are not part
// of the set until they are committed; cap[k] entries fit.
struct Lists {
    enum { VERTS, NORMALS, COLORS, VALUES, CONFS, PIX, N_LISTS };
    static constexpr int PER[N_LISTS] = {3, 3, 4, 1, 1, 2};
    bool on_device = false;
    void* p[N_LISTS] = {};
    uint64_t n[N_LISTS] = {}, staged[N_LISTS] = {}, cap[N_LISTS] = {};
};

// The points of one reference view until the call commits them: [at[k], at[k] + count[k]) of list k, staged
struct Block {
    b200mvs_pset_view rec = {0, 0.f, 0, 0};          // first_index is set by commit
    uint64_t at[Lists::N_LISTS] = {}, count[Lists::N_LISTS] = {};
    uint32_t view_id = 0, width = 0, height = 0;
    double ms_pointset = 0, ms_filter = 0;
};

// The device allocator of the handle's workspace while a reconstruction runs: the context's accounted one
struct Allocator {
    void* user = nullptr;
    cudaError_t (*alloc)(void* user, void** p, size_t bytes) = nullptr;
    void (*free)(void* user, void* p, size_t bytes) = nullptr;
};

// B200MVS_ERR_INVALID_ARG (message in b200mvs_last_error) for a NULL handle, a handle on another device than
// `device` or one whose masks have been applied
int check(const b200mvs_pset* ps, int device);
// Device bytes the handle's workspace holds at most for one map of w x h pixels with a colour image
uint64_t workspace_bytes(const b200mvs_pset* ps, int w, int h);
// Frees the workspace, then allocates it through `a` from here on (NULL: cudaMalloc)
void use_allocator(b200mvs_pset* ps, const Allocator* a);
// What b200mvs_pset_add_view does with the map and a 3-channel colour image, for a DEVICE depth map (w x h floats) and
// colours read in place from an RGBX level (uchar4, row pitch `pitch` texels); the points are staged, `out` records where
int extract(b200mvs_pset* ps, int view_id, const float* d_depth, int w, int h, const void* d_rgbx, int pitch,
            const b200mvs_pset_camera& cam, Block& out);
// Commits the staged blocks to the handle in their order; records[j] receives block j's record (records may be NULL).  On
// an error (the staged points could not be put in order) the set is as before the call.
int commit(b200mvs_pset* ps, const std::vector<Block>& blocks, b200mvs_pset_view* records);
// Forgets what extract staged since the last commit (a call that failed): the set is as before the call
void discard(b200mvs_pset* ps);

} // namespace b200mvs_pset_dev
