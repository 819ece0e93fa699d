"""Data-parallel training step, H100-native mirror of `Trainer.train_step` (fairseq/trainer.py:780-1097).

One process per GPU (torchrun / torch.distributed, backend nccl).  Per update:
  zero flat grads -> for each micro-batch: criterion forward + hand-written backward (kernels accumulate into
  the flat fp32 gradient buffer) -> ONE all-reduce over that buffer, whose 8-float tail carries
  [sample_size, ntokens, nsentences, loss] (replaces the reference's three collectives: stats float64
  all-reduce trainer.py:1411-1449, gradient all-reduce legacy_distributed_data_parallel.py:76-165 and the
  grad-norm consistency check trainer.py:1451-1488) -> esp_sumsq_f32 -> esp_adam_step, which reads
  1/sample_size and computes the clip coefficient on the device (trainer.py:918-953 semantics: grads are
  normalised by the global sample_size, clipped to clip_norm, Adam with fp32 master weights, bf16 params
  refreshed).  No host<->device synchronisation inside the step.
"""
import torch
import torch.distributed as dist

from . import lib as _lib
from . import ops as _ops


class Trainer:
    def __init__(self, model, criterion, lr_scheduler, adam_betas=(0.9, 0.98), adam_eps=1e-8, weight_decay=0.0,
                 clip_norm=2.0, process_group=None, use_cuda_graphs=False, bucket_frames=64, bucket_tokens=16,
                 max_graphs=128, reduce_dtype="bf16"):
        self.model = model
        self.criterion = criterion
        self.lr_scheduler = lr_scheduler
        self.betas, self.eps, self.weight_decay, self.clip_norm = adam_betas, adam_eps, weight_decay, clip_norm
        self.flat = model.flat
        self.flat.init_master()
        dev = self.flat.p16.device
        self._sumsq = torch.zeros(1, dtype=torch.float32, device=dev)
        self._gnorm = torch.zeros(1, dtype=torch.float32, device=dev)
        self.num_updates = 0
        self.pg = process_group
        self.world = dist.get_world_size(process_group) if dist.is_available() and dist.is_initialized() else 1
        self.rank = dist.get_rank(process_group) if self.world > 1 else 0
        # the hand-written backward assumes d(sum loss) = 1: the trainer is the one caller that guarantees it
        if hasattr(criterion, "unit_grad_output"):
            criterion.unit_grad_output = True
        self.last_stats = None
        # Gradient exchange dtype.  "bf16" = what the reference sends (fairseq --bf16: bf16 .grad tensors through
        # legacy_distributed_data_parallel.py:76-165), half the NVLink bytes of the fp32 flat buffer; the 8 logging /
        # normalisation scalars of the tail travel in a second, 32-byte fp32 all-reduce.  "fp32": one all-reduce of the
        # flat fp32 buffer including its tail.
        assert reduce_dtype in ("bf16", "fp32")
        self.reduce_dtype = reduce_dtype
        self._g16 = None
        # schedule scalars and the dropout seed live in device memory (written from a pinned staging buffer once
        # per update) so that a captured CUDA graph of the whole step can be replayed with fresh values
        self.use_cuda_graphs = use_cuda_graphs and dev.type == "cuda"
        self._hyper = torch.zeros(2, dtype=torch.float32, device=dev)      # [lr, step]
        self._seed = torch.zeros(1, dtype=torch.int64, device=dev)
        pin = dev.type == "cuda"
        self._hyper_host = torch.zeros(2, dtype=torch.float32, pin_memory=pin)
        self._seed_host = torch.zeros(1, dtype=torch.int64, pin_memory=pin)
        _ops.set_seed_tensor(self._seed)
        # CUDA graphs are keyed on BUCKETED shapes: waveform length padded to a multiple of `bucket_frames` feature
        # frames, target length to a multiple of `bucket_tokens`, SpecAugment descriptor counts to multiples of 4,
        # so real (every-batch-different) length distributions hit a small set of graphs; least-recently-used graphs
        # are dropped beyond `max_graphs`.
        self.bucket_frames, self.bucket_tokens, self.max_graphs = bucket_frames, bucket_tokens, max_graphs
        self._graphs, self._seen, self._pool = {}, {}, None
        self.graph_hits = self.graph_misses = 0

    def get_lr(self):
        return self.lr_scheduler.lr

    def _stage_scalars(self):
        lr = self.lr_scheduler.step_update(self.num_updates)
        self._hyper_host[0] = lr
        self._hyper_host[1] = float(self.num_updates + 1)
        # one dropout stream per (update, rank); micro-batches of an update are separated in _fwd_bwd
        self._seed_host[0] = (self.num_updates + 1) * 1000003 + self.rank * 7919
        self._hyper.copy_(self._hyper_host, non_blocking=True)
        self._seed.copy_(self._seed_host, non_blocking=True)

    def _fwd_bwd(self, samples):
        """Forward + hand-written backward of every micro-batch into the flat gradient buffer -- pure device work;
        this is the part captured in a CUDA graph per input shape."""
        model, flat = self.model, self.flat
        flat.zero_grad()
        tail = flat.tail
        enc = getattr(model, "encoder", model)
        for i, sample in enumerate(samples):
            if not sample:
                continue
            if hasattr(enc, "dropout_seed"):
                enc.dropout_seed = 1 + i  # update_freq > 1: every micro-batch draws its own masks
            loss, sample_size, log = self.criterion(model, sample)
            loss.backward()
            model.sync_torch_grads_()
            # logging scalars ride in the gradient buffer's tail
            tail[0] += sample_size
            tail[1] += log["ntokens"]
            tail[2] += log["nsentences"]
            tail[3] += log["loss"].float()

    def _reduce_and_update(self):
        """ONE collective (gradients + stats tail), then grad-norm + fused Adam reading lr/step/sample_size from device
        memory.  Kept outside the CUDA graph: the NCCL call stays an ordinary stream operation."""
        flat = self.flat
        if self.world > 1:
            if self.reduce_dtype == "bf16":
                if self._g16 is None:
                    self._g16 = torch.empty(flat.numel, dtype=torch.bfloat16, device=flat.g32.device)
                _ops.cast_f32_bf16(flat.grads, self._g16)
                w1 = dist.all_reduce(flat.tail, op=dist.ReduceOp.SUM, group=self.pg, async_op=True)
                dist.all_reduce(self._g16, op=dist.ReduceOp.SUM, group=self.pg)
                w1.wait()
                _ops.cast_bf16_f32(self._g16, flat.grads)
            else:
                dist.all_reduce(flat.g32, op=dist.ReduceOp.SUM, group=self.pg)
        _ops.sumsq(flat.grads, self._sumsq)
        _ops.adam_step(flat.p32, flat.m, flat.v, flat.grads, flat.p16, 0.0, self.betas[0], self.betas[1], self.eps,
                       self.weight_decay, 1, self._sumsq, denom_dev=flat.tail[0:1], clip_norm=self.clip_norm,
                       gnorm_out=self._gnorm, hyper_dev=self._hyper)

    def _step_body(self, samples):
        self._fwd_bwd(samples)
        self._reduce_and_update()

    # ---- shape bucketing -------------------------------------------------------------------------------------
    @staticmethod
    def _round_up(n, m):
        return (n + m - 1) // m * m

    def _bucket_shapes(self, sample):
        """Padded ("bucket") shapes of one micro-batch: {net_input key or 'target': shape}."""
        ni = sample["net_input"]
        shapes = {}
        for k, v in ni.items():
            if not (torch.is_tensor(v) and v.is_cuda):
                continue
            shp = list(v.shape)
            if k == "src_tokens":
                if v.dim() == 2:    # raw waveform [B, N]: N -> samples of the next multiple of bucket_frames frames
                    frames = 1 + max(shp[1] - 400, 0) // 160
                    shp[1] = max(shp[1], 400 + (self._round_up(frames, self.bucket_frames) - 1) * 160)
                elif v.dim() == 3:  # features [B, T, F]
                    shp[1] = self._round_up(shp[1], self.bucket_frames)
            elif k in ("freq_masks", "time_masks"):
                shp[1] = self._round_up(shp[1], 4)
            elif k == "time_warp":  # [B, 2]: one (w0, w) per utterance, fixed shape
                pass
            elif k == "prev_output_tokens":
                shp[1] = self._round_up(shp[1], self.bucket_tokens)
            shapes[k] = tuple(shp)
        t = list(sample["target"].shape)
        if len(t) == 2:
            t[1] = self._round_up(t[1], self.bucket_tokens)
        shapes["target"] = tuple(t)
        return shapes

    def _has_pads(self, sample, shapes):
        """The predicate the model bakes into the captured kernels' arguments (length masking on/off): any utterance
        shorter than the (bucketed) encoder time axis, evaluated AFTER the conv front's subsampling."""
        ni = sample["net_input"]
        lens = ni["src_lengths_cpu"]
        T = shapes["src_tokens"][1]
        if len(shapes["src_tokens"]) == 2:
            lens = _ops.num_frames(lens)
            T = _ops.num_frames(T)
        out = self.model.output_lengths(lens)
        Tp = int(self.model.output_lengths(torch.tensor([T]))[0])
        return bool((out < Tp).any())

    def _signature(self, sample):
        shapes = self._bucket_shapes(sample)
        sig = [("pads", self._has_pads(sample, shapes))]
        sig += [(k, shapes[k], str(sample["net_input"][k].dtype)) for k in sorted(shapes) if k != "target"]
        sig.append(("target", shapes["target"]))
        return tuple(sig), shapes

    def _pad_value(self, key):
        if key in ("target", "prev_output_tokens"):
            return getattr(self.criterion, "pad_idx", getattr(self.criterion, "padding_idx", 1))
        return 0  # waveform samples / feature frames beyond src_lengths are never read; width-0 masks are no-ops

    def _fill_static(self, static, sample):
        for k, v in list(sample["net_input"].items()) + [("target", sample["target"])]:
            if not (torch.is_tensor(v) and v.is_cuda):
                continue
            dst = static["target"] if k == "target" else static["net_input"][k]
            if dst.shape == v.shape:
                dst.copy_(v, non_blocking=True)
            else:
                if k != "src_tokens" or v.dim() != 2:
                    # token / descriptor / feature-frame tails carry meaning (pad symbol, no-op mask, zero frames as
                    # collate_frames pads them); only raw-waveform samples beyond src_lengths are never read
                    dst.fill_(self._pad_value(k))
                dst[tuple(slice(0, n) for n in v.shape)].copy_(v, non_blocking=True)

    def _graphed_step(self, sample):
        key, shapes = self._signature(sample)
        entry = self._graphs.get(key)
        if entry is None:
            self.graph_misses += 1
            static = self._seen.get(key)
            if static is None:
                # first sight of this bucket: a plain eager step ON THE BUCKET-SHAPED buffers, so that every
                # shape-dependent cache (position tables, workspaces, kernel attributes) exists before capture
                ni = sample["net_input"]
                static = {"net_input": {k: (torch.full(shapes[k], self._pad_value(k), dtype=v.dtype, device=v.device)
                                            if k in shapes else v) for k, v in ni.items()},
                          "target": torch.full(shapes["target"], self._pad_value("target"), dtype=sample["target"].dtype,
                                               device=sample["target"].device)}
                self._seen[key] = static
                self._fill_static(static, sample)
                self._step_body([static])
                return
            del self._seen[key]
            self._fill_static(static, sample)
            graph = torch.cuda.CUDAGraph()
            torch.cuda.synchronize()
            n0 = _lib.launch_count()
            with torch.cuda.graph(graph, pool=self._pool):
                self._fwd_bwd([static])
            n_kernels = _lib.launch_count() - n0  # native kernels recorded in this graph
            _lib.load().esp_note_graph_replay(-n_kernels)  # capture itself executed nothing
            if self._pool is None:
                self._pool = graph.pool()
            entry = [graph, static, n_kernels, 0]
            self._graphs[key] = entry
            if len(self._graphs) > self.max_graphs:  # drop the least recently used graph
                old = min((k for k in self._graphs if k != key), key=lambda k: self._graphs[k][3])
                del self._graphs[old]
        else:
            self.graph_hits += 1
        graph, static, n_kernels, _ = entry
        entry[3] = self.num_updates
        self._fill_static(static, sample)
        # host-side lengths are not part of the graph, but the model reads them while CAPTURING only
        graph.replay()
        _lib.load().esp_note_graph_replay(n_kernels)
        self._reduce_and_update()

    def train_step(self, samples):
        """samples: list of micro-batches (update_freq entries); an empty dict is a dummy batch whose
        contribution is zero but which still joins the collective (trainer.py:1305-1313).

        With use_cuda_graphs, single-micro-batch updates are captured per input shape (second occurrence) and
        replayed afterwards: the ~1200 kernel launches of a step cost one graph launch on the host."""
        model = self.model
        model.train()
        model.set_num_updates(self.num_updates)
        self._stage_scalars()
        streaming = getattr(getattr(model, "encoder", None), "has_attn_mask", False)  # masks change per update: eager
        if (self.use_cuda_graphs and not streaming and len(samples) == 1 and samples[0]
                and "src_lengths_cpu" in samples[0]["net_input"]):
            self._graphed_step(samples[0])
        else:
            self._step_body(samples)
        self.num_updates += 1
        self.last_stats = self.flat.tail  # device tensor; read it lazily (e.g. every log_interval updates)
        return self.last_stats

    def stats(self):
        """Host copy of the last update's global stats (one sync; call at log intervals only)."""
        t = self.last_stats.detach().cpu().tolist()
        return {"sample_size": t[0], "ntokens": t[1], "nsentences": t[2], "loss": t[3], "gnorm": float(self._gnorm.item()),
                "lr": self.get_lr(), "num_updates": self.num_updates}
