"""Worker of tests/test_sharded_volumes.py::test_ranks_nccl_volumes_arrays_and_alpha_windows (and a manual check under torchrun):
slab mode and batch mode over NCCL for volumes, texture arrays and alpha-scale, against the single-GPU payloads, and the bytes
every rank uploads.
    python -m torch.distributed.run --nproc-per-node N tests/sharded_volumes_worker.py <outdir>"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

TILE = 32


def slab(rows, world, g):
    return rows * g // world, rows * (g + 1) // world


def expected_h2d(img, cfg, world, rank):
    """Bytes rank `rank` uploads in slab mode: the slices of its layers (3D block sizes), or per touched slice the rows of its
    part, widened to the pre-pass window with alpha-scale."""
    d, h, w = img.shape[:3]
    bx, by, bz = cfg.block_x, cfg.block_y, max(1, cfg.block_z)
    blocks_y = (h + by - 1) // by
    layers = (d + bz - 1) // bz if bz > 1 else d
    r0, r1 = slab(blocks_y * layers, world, rank)
    if r1 == r0:
        return 0
    slice_bytes = img[0].nbytes
    row_bytes = slice_bytes // h
    if bz > 1:
        return (min((r1 + blocks_y - 1) // blocks_y * bz, d) - r0 // blocks_y * bz) * slice_bytes
    total = 0
    for s in range(r0 // blocks_y, (r1 + blocks_y - 1) // blocks_y):
        a, b = max(r0, s * blocks_y) - s * blocks_y, min(r1, (s + 1) * blocks_y) - s * blocks_y
        y0, y1 = a * by, min(b * by, h)
        if cfg.a_scale_radius:
            r = cfg.a_scale_radius
            y0, y1 = max(0, y0 // TILE * TILE - r), min(h, (y1 + TILE - 1) // TILE * TILE + r)
        total += (y1 - y0) * row_bytes
    return total


def main():
    import torch
    import torch.distributed as dist
    import astc_images as I
    from __graft_entry__ import load_package
    pkg = load_package()
    rank = int(os.environ["RANK"])
    world = int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")          # only to ship the NCCL id: the payload gather is the library's own NCCL
    box = [pkg.comm_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(box, src=0)
    S = pkg.FLG_SELF_DECOMPRESS_ONLY
    vol = lambda d, h, w, seed: np.stack([I.photo_like(h, w, seed=seed + z) for z in range(d)])  # noqa: E731
    # (config, images for slab mode): borders inside a layer / a slice, more ranks than combined rows, alpha-scale off the grid
    cases = [
        (pkg.config_init(pkg.PRF_LDR, 4, 4, pkg.PRE_MEDIUM, S, block_z=4), [vol(10, 37, 29, 1), vol(4, 4, 8, 2), vol(1, 30, 19, 3)]),
        (pkg.config_init(pkg.PRF_LDR, 5, 4, pkg.PRE_FASTEST, S, block_z=3), [vol(11, 23, 26, 4)]),
        (pkg.config_init(pkg.PRF_LDR, 6, 6, pkg.PRE_MEDIUM, S), [vol(3, 20, 40, 5), vol(5, 7, 30, 6), vol(2, 6, 6, 7)]),
        (pkg.config_init(pkg.PRF_LDR, 6, 6, pkg.PRE_FAST, S | pkg.FLG_USE_ALPHA_WEIGHT, a_scale_radius=8), [I.alpha_mask(250, 200, seed=8)[None],
                                                                                                      I.alpha_mask(9, 70, seed=9)[None]]),
    ]
    ok = True
    for cfg, imgs in cases:
        ctx = pkg.Context(cfg)
        ctx.comm_init(rank, world, box[0])
        solo = pkg.Context(cfg) if rank == 0 else None
        for img in imgs:
            got = ctx.compress_image_sharded(img)
            h2d = ctx.last_timing()[1]
            want_h2d = expected_h2d(img, cfg, world, rank)
            if h2d != want_h2d:
                print("rank %d: %s uploaded %d bytes, expected %d" % (rank, img.shape, h2d, want_h2d), flush=True)
                ok = False
            if rank == 0 and not np.array_equal(got, solo.compress_image(img)):
                print("slab mode differs from one GPU: %s block %dx%dx%d" % (img.shape, cfg.block_x, cfg.block_y, cfg.block_z), flush=True)
                ok = False
        # batch mode: image i on rank i % world, a ragged last round
        n = 2 * world + 1
        base = imgs[0]
        imgs_all = [np.ascontiguousarray(np.roll(base, 3 * i, axis=2)) for i in range(n)]
        mine = [imgs_all[i] if i % world == rank else None for i in range(n)]
        outs = None
        if rank == 0:
            outs = [np.zeros_like(solo.compress_image(imgs_all[0])) for _ in range(n)]
        ctx.compress_batch(mine, outs)
        if rank == 0:
            for i in range(n):
                if not np.array_equal(outs[i], solo.compress_image(imgs_all[i])):
                    print("batch mode differs from one GPU: image %d of %s" % (i, base.shape), flush=True)
                    ok = False
            solo.close()
        ctx.close()
    flags = [None] * world
    dist.all_gather_object(flags, ok)
    dist.destroy_process_group()
    if rank == 0 and all(flags) and len(sys.argv) > 1:
        open(os.path.join(sys.argv[1], "ok"), "w").write("ok\n")
    if not all(flags):
        sys.exit(1)


if __name__ == "__main__":
    main()
