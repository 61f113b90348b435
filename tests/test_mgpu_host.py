"""Host-side logic of the z-slab mode on CPU: partitions cover everything exactly once, and the control-plane exchange works
with world_size 2 over gloo (the data path itself needs GPUs: tools/mgpu_check.py under torchrun)."""
import os
import subprocess
import sys

import numpy as np

from conftest import ROOT


def test_partitions_cover_exactly_once():
    from kintinuous_b200 import mgpu
    for vol in (256, 512, 1024):
        for world in (1, 2, 4, 8):
            for block in (1, 4, 8, 16):
                owned = np.zeros(vol, int)
                for r in range(world):
                    planes = mgpu.owned_planes(r, world, vol, block)
                    assert len(planes) == vol // world
                    for l, z in enumerate(planes):
                        owned[z] += 1
                        assert mgpu.owner_of_plane(z, world, block) == r and mgpu.local_plane(z, world, block) == l
                assert (owned == 1).all()
                # balance: any window of block * world consecutive storage planes holds exactly `block` planes of every rank
                for r in range(world):
                    mine = np.zeros(vol, int); mine[mgpu.owned_planes(r, world, vol, block)] = 1
                    w = block * world
                    assert all(mine[s:s + w].sum() == block for s in range(0, vol, w))
    for rows in (480, 960, 120):
        for world in (1, 2, 4, 8):
            cover = np.zeros(rows // 8, int)
            for r in range(world):
                a, b = mgpu.tile_rows(r, world, rows)
                cover[a:b] += 1
            assert (cover == 1).all()


WORKER = r'''
import os, sys
sys.path.insert(0, sys.argv[1])
import torch.distributed as dist
from kintinuous_b200 import mgpu
dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
handle = bytes([rank]) * 64                      # stands in for the 64-byte cudaIpcMemHandle_t
got = mgpu.exchange(handle)
assert len(got) == world and all(got[r] == bytes([r]) * 64 for r in range(world)), got
n_mine = len(mgpu.owned_planes(rank, world, 512, 8))
import torch
t = torch.tensor([n_mine], dtype=torch.int64)
dist.all_reduce(t)
assert int(t.item()) == 512
dist.barrier()
print("rank", rank, "ok")
'''


def test_control_plane_world2_gloo(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port", "29533",
                          str(script), ROOT], capture_output=True, text=True, env=env, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.count("ok") == 2


def test_split_icp_pixel_partition_covers_every_pixel_once():
    """KT_MG_SPLIT_ICP: world * 132 CTAs (one per H100 SM) split the pixels of every pyramid level; the ranges must tile [0, N) exactly and
    be 4-pixel aligned (the TMA bulk copies need 16-byte granules).  The host stages min(passes, STAGE_MAX_K = 18) passes of a range
    (kt_icp.cu): 18 passes must fit an H100 block's 227 KB beside the kernel's static shared memory, and only level 0 of 1280x960 on one
    GPU (19 passes) streams a remainder from global memory."""
    from kintinuous_b200 import mgpu
    for rows, cols in ((480, 640), (960, 1280)):
        for level in range(3):
            n = (rows >> level) * (cols >> level)
            for world in (1, 2, 4, 8):
                ctas = 132
                seen = 0
                worst = 0
                for rank in range(world):
                    for cta in range(ctas):
                        b, c = mgpu.icp_pixel_range(rank, world, cta, ctas, n)
                        assert b == min(n, seen) and c >= 0 and b % 4 == 0
                        seen += c
                        worst = max(worst, c)
                assert seen == n
                # the stage holds min(ceil(q / 512), 18) passes of 512 pixels x 6 planes x 4 bytes
                passes = -(-worst // 512)
                assert min(passes, 18) * 512 * 6 * 4 <= 227 * 1024 - 4096
                assert (passes > 18) == ((rows, cols, level, world) == (960, 1280, 0, 1)), (rows, level, world, passes)
