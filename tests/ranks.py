"""Running a test across ranks, with every rank reaped however the test ends.

run_ranks launches a tests/mgpu_*_check.py script under torchrun and checks the line its rank 0 prints; init_rank and
finish_rank are that script's setup and teardown. spawn_ranks runs a function on in-process gloo ranks on the CPU.

torchrun starts each rank in a session of its own, so killing torchrun's process group does not reach the ranks, and a
rank left running holds its GPU memory. run_ranks therefore kills the whole process tree below torchrun, on every exit
path."""
import os
import queue
import signal
import socket
import subprocess
import sys
import time

import pytest

TESTS = os.path.dirname(os.path.abspath(__file__))


# ------------------------------------------------------------------------------------------------ torchrun ranks
def _descendants(pid):
    """The pids of every process below `pid`, from /proc."""
    children = {}
    for entry in os.listdir("/proc"):
        if entry.isdigit():
            try:
                with open("/proc/%s/stat" % entry) as f:
                    ppid = int(f.read().rsplit(")", 1)[1].split()[1])   # the command name may hold spaces
            except (OSError, IndexError, ValueError):   # the process has exited meanwhile
                continue
            children.setdefault(ppid, []).append(int(entry))
    found, todo = [], [pid]
    while todo:
        kids = children.get(todo.pop(), [])
        found += kids
        todo += kids
    return found


def _kill_tree(p, grace=10.0):
    """SIGKILL torchrun (started in a new session, so its pid is its process group's id) and every process below it,
    then wait for torchrun and, for up to `grace` seconds, for the others to be gone."""
    if p.poll() is not None:
        return
    os.killpg(p.pid, signal.SIGSTOP)   # no new rank can start while the tree is read
    pids = _descendants(p.pid)
    os.killpg(p.pid, signal.SIGKILL)
    for pid in pids:
        try:
            os.kill(pid, signal.SIGKILL)
        except ProcessLookupError:
            pass
    p.wait()
    deadline = time.monotonic() + grace
    for pid in pids:
        while time.monotonic() < deadline:
            try:
                os.kill(pid, 0)
            except ProcessLookupError:
                break
            time.sleep(0.05)


def run_ranks(script, sentinel, timeout):
    """Run tests/<script> under torchrun with 4 ranks on a machine with four or more GPUs, else 2, and assert that it
    exits with 0 and prints `sentinel`. On a timeout, an exception or an interrupt, torchrun and every rank are killed
    before this returns."""
    import torch

    world = 4 if torch.cuda.device_count() >= 4 else 2
    cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc-per-node", str(world),
           os.path.join(TESTS, script)]
    p = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, start_new_session=True)
    try:
        try:
            out, err = p.communicate(timeout=timeout)
        except subprocess.TimeoutExpired:
            _kill_tree(p)
            out, err = p.communicate()
            pytest.fail("%s timed out: %s%s" % (script, out[-2000:], err[-2000:]))
    finally:
        _kill_tree(p)
    assert p.returncode == 0 and sentinel in out, out[-3000:] + err[-3000:]


def init_rank():
    """Join the torchrun process group: (rank, world, device, context). With fewer GPUs than ranks every rank runs on
    GPU 0 and the ranks exchange through gloo, since NCCL refuses two ranks on one device; otherwise rank r runs on
    GPU LOCAL_RANK over NCCL."""
    import torch
    import torch.distributed as dist

    import plonky2_b200 as pb

    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    shared = torch.cuda.device_count() < world
    dev = torch.device("cuda", 0 if shared else local)
    torch.cuda.set_device(dev)
    if shared:
        dist.init_process_group("gloo")
    else:
        dist.init_process_group("nccl", device_id=dev)
    return rank, world, dev, pb.default_context(dev.index)


def finish_rank(name, failures, **info):
    """Gather every rank's failures; rank 0 prints "<name> OK|FAILED world <n> backend <b>", each `info` item and the
    failures. Then leave the process group and exit, with 1 on every rank if any rank failed."""
    import torch.distributed as dist

    everyone = [None] * dist.get_world_size()
    dist.all_gather_object(everyone, failures)
    ok = not any(everyone)
    if dist.get_rank() == 0:
        print(name, "OK" if ok else "FAILED", "world", dist.get_world_size(), "backend", dist.get_backend(),
              *[x for item in info.items() for x in item], [f for fs in everyone for f in fs], flush=True)
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


# ---------------------------------------------------------------------------------------------- CPU gloo ranks
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _rank_main(target, rank, world, port, args, results):
    import torch.distributed as dist

    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % port, rank=rank, world_size=world)
    try:
        results.put((rank, target(rank, world, *args)))
    finally:
        dist.destroy_process_group()


def spawn_ranks(target, world, args=(), timeout=180):
    """target(rank, world, *args) on `world` spawned processes joined in a gloo process group: the list of what each
    rank returned, in rank order. Every rank must return and exit with 0 within `timeout` seconds. However this ends,
    ranks still alive are terminated, then killed."""
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    results = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_rank_main, args=(target, r, world, port, args, results)) for r in range(world)]
    deadline = time.monotonic() + timeout
    started = []
    try:
        for p in procs:
            p.start()
            started.append(p)
        got = {}
        while len(got) < world:
            try:
                rank, value = results.get(timeout=1)
                got[rank] = value
            except queue.Empty:
                failed = [(r, p.exitcode) for r, p in enumerate(procs) if p.exitcode not in (None, 0)]
                assert not failed, "ranks exited before returning: (rank, exit code) %s" % failed
                assert time.monotonic() < deadline, "ranks %s did not return within %d s" % (
                    sorted(set(range(world)) - set(got)), timeout)
        for p in procs:
            p.join(max(0.0, deadline - time.monotonic()))
        assert [p.exitcode for p in procs] == [0] * world, "exit codes %s" % [p.exitcode for p in procs]
        return [got[r] for r in range(world)]
    finally:
        for p in started:
            if p.is_alive():
                p.terminate()
        for p in started:
            p.join(5)
            if p.is_alive():
                p.kill()
                p.join()
