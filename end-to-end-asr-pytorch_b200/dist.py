"""Data parallelism over the 8 GPUs of one box: one process per GPU (torchrun), utterances of the GLOBALLY sorted and
GLOBALLY padded batch sharded across ranks, ONE NCCL all-reduce(sum) of the flat fp32 gradient buffer per step.

The reference has no distributed code at all (SURVEY.md 2.1); the rules that keep a DP step identical to the
reference's single-process step are (SURVEY.md 8(e)):
  * pad to the global T_max / decode to the global max(txt_len) - the encoder runs through the padding (F5);
  * CTC 'mean': each rank back-props sum_b nll_b / len_b / B_global; CE: sum over its tokens / N_tok_global;
  * all-reduce = SUM, then every rank computes the identical global grad-norm, clip and update.
"""
import os

import torch
import torch.distributed as dist


class DataParallel:
    def __init__(self, backend=None):
        self.world = int(os.environ.get("WORLD_SIZE", "1"))
        self.rank = int(os.environ.get("RANK", "0"))
        self.local_rank = int(os.environ.get("LOCAL_RANK", "0"))
        self.enabled = self.world > 1
        self.backend = backend
        if self.enabled and not dist.is_initialized():
            if backend is None:
                backend = "nccl" if torch.cuda.is_available() else "gloo"
            os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
            os.environ.setdefault("MASTER_PORT", "29500")
            if backend == "nccl":
                torch.cuda.set_device(self.local_rank)
                # The LSTM step kernels are cooperative: 128 CTAs, one per SM, all co-resident - 4 of the 132 SMs stay
                # free.  An all-reduce with more CTAs than that cannot run NEXT to them, so the exchange of a layer's
                # gradients serialises with the next layer's backward instead of hiding behind it.  4 follows from the SM
                # count alone: its cost in all-reduce bandwidth has not been measured.
                os.environ.setdefault("NCCL_MAX_CTAS", "4")
            dist.init_process_group(backend=backend, rank=self.rank, world_size=self.world)
            self.backend = backend

    @classmethod
    def single(cls):
        """A disabled communicator (world 1) regardless of the torchrun environment: the single-GPU reference of a
        data-parallel step."""
        o = cls.__new__(cls)
        o.world, o.rank, o.enabled, o.backend = 1, 0, False, None
        o.local_rank = int(os.environ.get("LOCAL_RANK", "0"))
        return o

    def shard(self, *tensors):
        """Rank r takes rows r::world of each [B_global, ...] tensor (lengths sorted desc => equal work)."""
        if not self.enabled:
            return tensors if len(tensors) > 1 else tensors[0]
        out = tuple(t[self.rank::self.world].contiguous() for t in tensors)
        return out if len(out) > 1 else out[0]

    def all_reduce_(self, flat, n_buckets=1):
        """In-place SUM of the flat gradient buffer (bucketed so later buckets overlap earlier ones' epilogue)."""
        if not self.enabled:
            return flat
        if n_buckets <= 1:
            dist.all_reduce(flat, op=dist.ReduceOp.SUM)
            return flat
        n = flat.numel()
        step = (n + n_buckets - 1) // n_buckets
        works = [dist.all_reduce(flat[i:i + step], op=dist.ReduceOp.SUM, async_op=True) for i in range(0, n, step)]
        for w in works:
            w.wait()
        return flat

    def all_reduce_scalar(self, value, device):
        if not self.enabled:
            return value
        t = torch.tensor([float(value)], device=device, dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.SUM)
        return float(t.item())

    def max_time(self, ms, device):
        """Max over ranks of a per-rank duration (multi-GPU numbers are the slowest rank's)."""
        if not self.enabled:
            return ms
        t = torch.tensor([float(ms)], device=device, dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    def barrier(self):
        if self.enabled:
            dist.barrier()

    def attach(self, optimizer, model=None):
        """Make the gradient exchange part of the step.

        With `model`: the flat gradient buffer is cut into per-layer BUCKETS (every encoder layer; everything after the
        encoder - CTC head, embedding, decoder, attention - is one bucket) and each bucket's NCCL all-reduce is launched
        from a post-accumulate hook the moment the LAST gradient of that bucket has been written by autograd.  The
        backward pass produces the decoder / attention / CTC-head gradients first and the encoder layers top-down, so
        all but the first encoder layer's exchange overlaps the rest of the backward (SURVEY.md 8(e)).
        `optimizer.step()` launches whatever has not fired (parameters without gradients) and waits for all of them.
        Without `model`: one all-reduce of the whole buffer inside `optimizer.step()`."""
        if not self.enabled:
            return optimizer
        if model is None:
            optimizer.pre_reduce = lambda flat: self.all_reduce_(flat, 1)
            return optimizer
        buf = optimizer.buf
        index = {id(p): i for i, p in enumerate(buf.params)}
        groups = {}
        for name, p in model.named_parameters():
            if id(p) not in index:
                continue
            parts = name.split(".")
            key = ".".join(parts[:3]) if parts[0] == "encoder" else "head"
            groups.setdefault(key, []).append(index[id(p)])
        self._buckets = []
        for key, ids in groups.items():
            ids.sort()
            lo = buf.offsets[ids[0]]
            hi = buf.offsets[ids[-1]] + (buf.params[ids[-1]].numel() + 3) // 4 * 4
            self._buckets.append({"key": key, "ids": set(ids), "lo": lo, "hi": hi, "seen": 0, "work": None})
        # the buckets must tile the buffer (parameters are registered module by module)
        self._buckets.sort(key=lambda b: b["lo"])
        pos = 0
        for b in self._buckets:
            assert b["lo"] == pos, "gradient buckets are not contiguous: %s" % b["key"]
            pos = b["hi"]
        assert pos == buf.total
        by_param = {}
        for b in self._buckets:
            for i in b["ids"]:
                by_param[i] = b

        def launch(b):
            # after close() (communicator torn down) the hooks degrade to the single-process behaviour: rank 0 may keep
            # stepping on its own shard, e.g. bench.py's parity block after the timed regions
            if b["work"] is None and self.enabled and dist.is_initialized():
                b["work"] = dist.all_reduce(buf.grad[b["lo"]:b["hi"]], op=dist.ReduceOp.SUM, async_op=True)

        def make_hook(i):
            b = by_param[i]

            def hook(param):
                # autograd may have replaced .grad by a fresh tensor: fold it back into the flat buffer first
                o = buf.offsets[i]
                if param.grad is not None and param.grad.data_ptr() != buf.grad.data_ptr() + 4 * o:
                    view = buf.grad[o:o + param.numel()].view(param.shape)
                    view.copy_(param.grad)
                    param.grad = view
                b["seen"] += 1
                if b["seen"] == len(b["ids"]):
                    launch(b)
            return hook

        for i, p in enumerate(buf.params):
            p.register_post_accumulate_grad_hook(make_hook(i))

        def finish(flat):
            for b in self._buckets:
                launch(b)
            for b in self._buckets:
                if b["work"] is not None:
                    b["work"].wait()
                b["work"], b["seen"] = None, 0
            return flat

        optimizer.pre_reduce = finish
        return optimizer

    def close(self):
        """Tear the communicator down (call before interpreter exit: NCCL warns - and can hang - otherwise)."""
        if self.enabled and dist.is_initialized():
            dist.barrier()
            dist.destroy_process_group()
            self.enabled = False
