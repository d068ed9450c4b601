"""Worker of tests/test_sharded_handel_gloo.py (TEST INFRASTRUCTURE): one node-id shard of a Handel network per process over
gloo (DistributedHandel: the handles of the exchange regions travel once through torch.distributed, the data path is stores
into the peers' regions).  The simulation runs on the host build of the device logic (tests/emu), whose exchange regions are
POSIX shared memory where the CUDA backend uses CUDA IPC."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch.distributed as dist  # noqa: E402

from tests import emu_handel_lib as emu_lib  # noqa: E402
from tests.parity import handel_digests  # noqa: E402
from wittgenstein_b200 import HandelParameters  # noqa: E402
from wittgenstein_b200.sharded import DistributedHandel  # noqa: E402

dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()

# Handel, 256 nodes, 64 suicide-Byzantine: this rank owns ids [rank * 128, rank * 128 + 128)
prm = HandelParameters(256, 153, 4, 50, 10, 20, 10, 64, "AWS_SPEED=GAUSSIAN_TOR=0.33", "AwsRegionNetworkLatency", 0, True, False)
p = DistributedHandel(prm, dist, rank, world, None, _api=emu_lib.api())
p.init()
digests = {}
while p.continue_if() and p.network().time < 4000:
    p.network().run_ms(50)
    if p.network().time % 250 == 0:
        digests[p.network().time] = handel_digests(p.local, False)
net = p.network()
out = {"rank": rank, "range": list(net.shard_range()), "time": net.time, "digests": digests}
print("RANKLINE " + json.dumps(out), flush=True)
dist.barrier()
dist.destroy_process_group()
