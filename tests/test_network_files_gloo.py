"""World-size-2 run of inference_combined's host side on CPU (gloo): each rank takes its DistributedSampler(shuffle=False)
shard of the test scenes, records per-scene metrics in InferenceMetrics, and rank 0 gathers them and writes the report,
which must equal the report written from the same records gathered by hand (the reference's gather_all_metrics)."""
import os
import socket
import sys

import pytest
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _scene_metrics(i):
    """Deterministic per-scene metrics; scenes 2k and 2k+1 belong to the same object."""
    v = (i * 0.137) % 1.0
    return f"obj{i // 2}", {"seg_acc": v, "density_mse": v / 3, "youngs_mse": v / 5, "poisson_mse": v / 7, "cont_mse": v / 4}


def _record(NF, scenes):
    m = NF.InferenceMetrics()
    for i in scenes:
        obj, s = _scene_metrics(i)
        m.add_batch_metrics(s["seg_acc"], s["cont_mse"], s["density_mse"], s["youngs_mse"], s["poisson_mse"])
        m.add_sample_metrics(obj, s)
        m.local_obj_ids.append(obj)
    return m


def _worker(rank, world, port, n_scenes, out_dir, q):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    from pixie_b200 import dist_utils as D, network_files as NF
    D.init("gloo")
    mine = D.shard_scenes(n_scenes, rank, world)
    gathered = _record(NF, mine).gather_all_metrics(rank, world)
    if rank == 0:
        NF.generate_metrics_report(gathered, out_dir, "seg.pth", "cont.pth", "sem")
    q.put((rank, mine))
    dist.destroy_process_group()


@pytest.mark.parametrize("n_scenes", [7, 8])
def test_sharded_report_matches_single_rank(tmp_path, n_scenes):
    sys.path.insert(0, ROOT)
    from torch.utils.data import DistributedSampler
    from pixie_b200 import network_files as NF
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    (tmp_path / "dist").mkdir()
    procs = [ctx.Process(target=_worker, args=(r, world, port, n_scenes, str(tmp_path / "dist"), q)) for r in range(world)]
    for p in procs:
        p.start()
    shards = dict(q.get(timeout=120) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for r in range(world):
        assert shards[r] == list(DistributedSampler(range(n_scenes), num_replicas=world, rank=r, shuffle=False))
    # the reference's gather: one list per rank, in rank order
    per_rank = [_record(NF, shards[r]) for r in range(world)]
    lists = [[m.seg_accuracies for m in per_rank], [m.cont_mse_values for m in per_rank], [m.density_mse_values for m in per_rank],
             [m.youngs_mse_values for m in per_rank], [m.poisson_mse_values for m in per_rank], [m.local_obj_ids for m in per_rank],
             [m.obj_metrics for m in per_rank]]
    (tmp_path / "single").mkdir()
    NF.generate_metrics_report(lists, str(tmp_path / "single"), "seg.pth", "cont.pth", "sem")
    for f in ("metrics.json", "evaluated_obj_ids.json"):
        assert (tmp_path / "dist" / f).read_bytes() == (tmp_path / "single" / f).read_bytes()
