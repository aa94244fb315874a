"""Multi-GPU learner behind the reference's Trainer surface: one process per GPU, no torchrun needed.

The reference switches its multi-GPU mode on inside Trainer (nn.DataParallel when torch.cuda.device_count() > 1,
handyrl/train.py:325, 339-340), so `python main.py --train` just uses every GPU.  Here the Trainer's own process is
rank 0 (it hosts the Learner, the worker server and the epoch hand-off) and `Fleet` spawns one helper process per
further GPU.  Every rank holds the WHOLE replay (rank 0 forwards each arriving episode once; every helper decodes
and uploads it with its own feeder thread), draws batch_size / world windows per step from it with an independent
random stream -- the union is batch_size i.i.d. draws of the reference's sampling law, train.py:291-315 -- and runs
the captured step whose gradient bucket (with the loss sums and the data count in its tail) is all-reduced with SUM
(fused NVLink peer-memory kernel, or NCCL).  Clip threshold, Adam and the learning-rate schedule therefore see global
quantities (train.py:327-331, 370, 382-384) and stay bit-identical on all ranks without any broadcast.

Control: rank 0 tells the helpers how many steps to run ("run n": whole chunks, so that every rank executes exactly
the same number of collectives) and when an epoch ends ("epoch": the device-side learning-rate update).  Helpers never
hand a model back: rank 0's weights are everyone's weights.
"""
import os
import pickle
import queue
import random
import socket
import threading
import time
import traceback

import torch


def _free_port():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def pin_to_gpu_numa(device_index):
    """Restrict this process to the CPUs of the NUMA node the GPU hangs off (PCIe locality of pinned copies and of
    the launch path); returns the CPU list or None when the topology cannot be read."""
    try:
        pr = torch.cuda.get_device_properties(device_index)
        bdf = '%04x:%02x:%02x.0' % (pr.pci_domain_id, pr.pci_bus_id, pr.pci_device_id)
        with open('/sys/bus/pci/devices/%s/local_cpulist' % bdf) as f:
            spec = f.read().strip()
        cpus = set()
        for part in spec.split(','):
            if '-' in part:
                a, b = part.split('-')
                cpus.update(range(int(a), int(b) + 1))
            elif part:
                cpus.add(int(part))
        allowed = cpus & os.sched_getaffinity(0)
        if allowed:
            os.sched_setaffinity(0, allowed)
            return sorted(allowed)
    except Exception:
        return None
    return None


# ---- torchrun-launched ranks (bench.py, scripts): the same sharding, with the ranks created by the launcher

def init_from_env(backend=None):
    """Initialise torch.distributed from RANK / WORLD_SIZE / MASTER_* (torchrun); returns (rank, world, local)."""
    import torch.distributed as dist
    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = 'nccl' if torch.cuda.is_available() else 'gloo'
        kw = {}
        if backend == 'nccl':
            torch.cuda.set_device(local)
            kw['device_id'] = torch.device('cuda', local)
        dist.init_process_group(backend, **kw)
    return rank, world, local


def shard_bounds(B, rank, world):
    """Contiguous split of the batch dimension; the first B % world ranks get one extra window."""
    base, extra = divmod(B, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def shard_batch(batch, rank, world):
    """Slice every (B, ...) tensor of a make_batch dict (nested observations included) to this rank's windows."""
    from .batch import tree_map
    B = batch['action'].shape[0]
    lo, hi = shard_bounds(B, rank, world)
    return tree_map(lambda t: t[lo:hi].contiguous(), batch)


def allreduce_sum_(flat, group=None):
    """In-place SUM all-reduce of the flat gradient bucket (gradients + appended loss sums)."""
    import torch.distributed as dist
    if dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
    return flat


def _init_group(rank, world, port):
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl', init_method='tcp://127.0.0.1:%d' % port, rank=rank, world_size=world,
                            device_id=torch.device('cuda', rank))
    return dist.group.WORLD


def _helper_main(rank, world, port, args, model_blob, lr, conn, optim_state=None):
    """Body of a helper rank (own process, own GPU).  `optim_state`: the optimiser state rank 0 resumes from (an
    OptimizerStateFormat dict, replicated on every rank), or None."""
    try:
        from .train import Batcher, EpisodeDeque, GpuBatcher, LearnerStep
        from .batch import tree_map
        pin_to_gpu_numa(rank)
        random.seed(args.get('seed', 0) * 1000003 + rank)
        pg = _init_group(rank, world, port)
        device = torch.device('cuda', rank)
        model = pickle.loads(model_blob)
        episodes = EpisodeDeque()
        cmds = queue.Queue()

        def reader():
            while True:
                try:
                    msg = conn.recv()
                except (EOFError, OSError):
                    cmds.put(('stop',))
                    return
                if msg[0] == 'episodes':
                    episodes.extend(msg[1])
                    while len(episodes) > args['maximum_episodes']:      # train.py:476-483
                        episodes.popleft()
                else:
                    cmds.put(msg)

        threading.Thread(target=reader, daemon=True).start()
        assert cmds.get()[0] == 'start'                # the backlog has arrived in `episodes`
        batch = Batcher(args, episodes)._make()
        batch = tree_map(lambda t: t[:t.shape[0] // world].contiguous(), batch)
        # rank 0 averages, validates and writes the optimiser state
        stepper = LearnerStep(model, args, batch, lr, device=device, process_group=pg, weight_ema=0, save_optimizer=False,
                              validation=False)
        if optim_state is not None:
            stepper.load_optimizer_state(optim_state)
        stepper.warm_up()
        # rank 0 validates: the held-out episodes (the same ones on every rank) are left out here
        gb = GpuBatcher(args, episodes, device, seed=args.get('seed', 0) * 7919 + 17 + rank, keep_validation=False)
        gb.run()
        while not gb.ready():
            time.sleep(0.005)
        conn.send(('ready',))
        while True:
            cmd = cmds.get()
            if cmd[0] == 'run':
                for _ in range(cmd[1]):
                    gb.fill(stepper)
                    stepper.step_in_place()
            elif cmd[0] == 'epoch':
                with torch.cuda.stream(stepper.stream):
                    stepper.epoch_schedule(cmd[1], cmd[2], cmd[3])
                if cmd[4]:           # parity probe: checksum of the weights after the epoch's steps
                    stepper.stream.synchronize()
                    conn.send(('weights', stepper.state.flat_param.double().sum().item(),
                               float(stepper.opt.lr.item())))
            elif cmd[0] == 'stop':
                break
        gb.stop()
        stepper.close()
        import torch.distributed as dist
        dist.barrier()
        torch.cuda.synchronize()
        dist.destroy_process_group()
        conn.send(('bye',))
    except Exception:
        traceback.print_exc()
        try:
            conn.send(('error', traceback.format_exc()))
        except Exception:
            pass


class Fleet:
    """Rank 0's handle on the helper ranks.  `optim_state` (an OptimizerStateFormat dict, or None) is the optimiser state
    every helper loads before its first step."""

    def __init__(self, world, args, template, backlog, lr, optim_state=None):
        import torch.multiprocessing as mp
        self.world = world
        self.args = args
        ctx = mp.get_context('spawn')
        port = _free_port()
        blob = pickle.dumps(template)
        plain_args = {k: v for k, v in args.items()}
        self.conns, self.procs = [], []
        for r in range(1, world):
            parent, child = ctx.Pipe()
            p = ctx.Process(target=_helper_main, args=(r, world, port, plain_args, blob, lr, child, optim_state), daemon=True)
            p.start()
            self.conns.append(parent)
            self.procs.append(p)
        pin_to_gpu_numa(0)
        self.process_group = _init_group(0, world, port)
        self.sent = set()
        self.send_lock = threading.Lock()
        self.send_episodes(backlog)
        self._send(('start',))
        self._ready = [False] * len(self.conns)
        self.probe = bool(args.get('multi_gpu_probe', False))
        self.reports = []

    def _send(self, msg):
        with self.send_lock:
            for c in self.conns:
                c.send(msg)

    def send_episodes(self, eps):
        """Forward episodes to every helper exactly once (the replay feeder calls this for everything it uploads)."""
        fresh = [e for e in eps if id(e) not in self.sent]
        if not fresh:
            return
        self.sent.update(id(e) for e in fresh)
        if len(self.sent) > 4 * self.args['maximum_episodes'] + 1024:
            self.sent = set(id(e) for e in fresh)
        self._send(('episodes', fresh))

    def all_ready(self):
        for i, c in enumerate(self.conns):
            while not self._ready[i] and c.poll(0):
                msg = c.recv()
                if msg[0] == 'ready':
                    self._ready[i] = True
                elif msg[0] == 'error':
                    raise RuntimeError('helper rank %d failed:\n%s' % (i + 1, msg[1]))
        return all(self._ready)

    def run_steps(self, n):
        self._send(('run', int(n)))

    def end_epoch(self, batch_cnt, steps, default_lr):
        self._send(('epoch', int(batch_cnt), int(steps), float(default_lr), self.probe))

    def collect_reports(self, timeout=30.0):
        """(weights checksum, lr) of every helper for the last epoch (multi_gpu_probe=True)."""
        out = []
        for c in self.conns:
            if not c.poll(timeout):
                raise TimeoutError('no report from a helper rank')
            msg = c.recv()
            assert msg[0] == 'weights', msg
            out.append((msg[1], msg[2]))
        return out

    def stop(self):
        try:
            self._send(('stop',))
        except Exception:
            pass

    def destroy(self):
        import torch.distributed as dist
        try:
            dist.barrier()
            torch.cuda.synchronize()
            dist.destroy_process_group()
        except Exception:
            traceback.print_exc()
        for p in self.procs:
            p.join(timeout=20)
            if p.is_alive():
                p.terminate()
