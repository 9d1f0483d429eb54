"""Pure data parallelism for the training step (BASELINE.json: "NCCL allreduce over NVLink on the gradient
buckets only").  One process per GPU; samples are independent units, so the only exchange is the gradient
all-reduce.  The reference has no distributed code of its own - its examples delegate to `accelerate` (DDP),
train_text_only.py:105-128 - this is the CUDA-native equivalent on the engine's flat gradient buffer.

Buckets: the flat buffer is laid out in `named_parameters()` order (layer 0 first).  Backward finishes layers
from the last to the first, so after layer i's kernels are enqueued the slice holding layers >= i is final and is
all-reduced on a side stream while the remaining layers run (`Engine.backward(bucket_cb=...)`).
"""
from __future__ import annotations

import torch
import torch.distributed as dist


class AsyncScalar:
    """Device scalar -> host without stalling the training stream: the D2H copy runs on a side stream behind an event recorded where the
    scalar was produced, so `.value()` waits for THAT step only - not for work enqueued afterwards (a plain `.item()` is ordered behind
    everything already in the stream, i.e. behind the next step when losses are logged one step late)."""
    _side = None

    def __init__(self, t: torch.Tensor):
        if AsyncScalar._side is None:
            AsyncScalar._side = torch.cuda.Stream()
        ready = torch.cuda.Event()
        ready.record()
        self.host = torch.empty((), dtype = t.dtype).pin_memory()
        self.done = torch.cuda.Event()
        with torch.cuda.stream(AsyncScalar._side):
            AsyncScalar._side.wait_event(ready)
            self.host.copy_(t.detach().reshape(()), non_blocking = True)
            self.done.record()
        self._keep = t

    def value(self) -> float:
        self.done.synchronize()
        return self.host.item()


class _StepGraph:
    """A captured training step (forward + backward + fused Adam) for ONE shape signature of the ragged batch descriptor."""
    def __init__(self):
        self.graph = None
        self.meta = None          # static device buffer holding the int / float metadata
        self.layout = None
        self.lat = None           # static per-type latent matrices
        self.rb = None            # the descriptor object the graph was captured with (its .dev views point into `meta`)
        self.loss = None
        self.eager_steps = 0
        self.meta_stage = self.lat_stage = self.consumed = None


class DataParallelTrainer:
    def __init__(self, model, lr = 1e-3, betas = (0.9, 0.999), eps = 1e-8, weight_decay = 0., decoupled_weight_decay = False, overlap = True, cuda_graph = True, graph_multi_gpu = True,
                 max_grad_norm = None, ema_decay = None, bucket_mb = 25):
        self.model = model
        self.hp = dict(lr = lr, betas = betas, eps = eps, weight_decay = weight_decay, decoupled = decoupled_weight_decay)
        self.world = dist.get_world_size() if dist.is_initialized() else 1
        self.overlap = overlap and self.world > 1
        self.comm_stream = None
        self.bucket_bytes = int(bucket_mb * 2 ** 20)
        self._cpu_opt = None
        # the rest of the step the reference's example scripts run: clip_grad_norm_(max_grad_norm) before the optimizer, EMA after it
        self.max_grad_norm, self.ema_decay = max_grad_norm, ema_decay
        # CUDA graphs: a step whose descriptor has a shape signature seen twice before is captured once and replayed afterwards - the ~320
        # kernel launches of a step (8-9 ms of host time through ctypes) become one graph launch.  With several ranks the gradient
        # all-reduce (NCCL) is captured inside the graph, after the backward pass (set graph_multi_gpu = False for the eager,
        # bucket-overlapped path instead).
        self.cuda_graph = cuda_graph and (self.world == 1 or graph_multi_gpu)
        self._graphs = {}
        self._copy_stream = None
        self._synced = False

    def _sync_replicas(self, eng):
        """Replicas must start identical (what DDP / accelerate do at construction): rank 0's parameters and persistent buffers
        (incl. the random Fourier frequencies of the time embedding) are broadcast once."""
        if self._synced or self.world == 1:
            self._synced = True
            return
        dist.broadcast(eng.flat, 0)
        for b in self.model.buffers():
            if b.is_cuda and b.numel():
                dist.broadcast(b, 0)
        eng.mark_dirty()
        self._synced = True

    # ---- CUDA-graph replay of fixed-shape steps
    @staticmethod
    def _signature(rb, eng):
        return (rb.M, rb.B, rb.n_cond, rb.S, tuple(rb.type_rows), tuple(getattr(rb, n).shape[0] if getattr(rb, n) is not None else 0 for n in eng.META_NAMES), rb.total_tokens,
                tuple(rb.n_type_tokens), (rb.max_rope_pos + 1 + 1023) // 1024, rb.has_labels, rb.pos_max)

    def _graph_step(self, rb, device_lat = None, noise = None, dropout_key = None):
        """Returns the loss of a replayed (or freshly captured) step, or None when this batch must run eagerly.
        device_lat: per-type latent matrices already on the device (then rb must be uploaded too: a device-resident batch)."""
        model, eng = self.model, self.model.engine
        drop = model.transformer.ff_dropout_p(True, model.training) > 0.
        recon = bool(model.has_recon_loss)
        sig = self._signature(rb, eng) + (drop, recon)     # a step with dropout / the reconstruction loss launches other kernels than one without
        g = self._graphs.get(sig)
        if g is None:
            if len(self._graphs) >= 8:
                return None
            g = self._graphs[sig] = _StepGraph()
        if g.graph is None and g.eager_steps < 2:       # let the buffers, weight packs and Adam state of this shape settle first
            g.eager_steps += 1
            return None
        # Stage this batch's inputs.  The host -> device copies run on a copy stream into staging buffers, so the PCIe transfer of step i+1
        # overlaps the graph of step i; a device-to-device copy (a few microseconds) moves them into the graph's static inputs.
        if device_lat is not None:
            src_meta = rb.dev['_keep']
            raw, host, layout = None, src_meta, rb.dev['_layout']
        else:
            raw, host, layout = eng.stage_meta(rb)
        if g.graph is None:
            g.meta = torch.empty_like(host, device = eng.device)
            g.meta_stage = torch.empty_like(g.meta)
            g.layout = layout
            g.lat = [torch.empty(s1 - s0, model.dim_latents[t], device = eng.device, dtype = torch.float32) if s1 > s0 else None for t, (s0, s1) in enumerate(rb.type_rows)]
            g.lat_stage = [torch.empty_like(l) if l is not None else None for l in g.lat]
            g.eps = [torch.empty_like(l) if l is not None else None for l in g.lat]      # flow noise: a static input of the graph, drawn (or injected) per step
            g.drop_key = torch.zeros(2, device = eng.device, dtype = torch.int32)     # dropout key: likewise
            g.consumed = torch.cuda.Event()
            g.consumed.record()
        assert layout == g.layout
        if device_lat is not None:                       # device-resident batch: plain device-to-device copies into the static inputs
            lat_bytes = 0
            g.meta.copy_(host, non_blocking = True)
            for dst, src in zip(g.lat, device_lat):
                if dst is not None:
                    dst.copy_(src, non_blocking = True)
        else:
            if self._copy_stream is None:
                self._copy_stream = torch.cuda.Stream()
            from ._pinned import POOL
            with torch.cuda.stream(self._copy_stream):
                self._copy_stream.wait_event(g.consumed)    # the previous step has moved the staging buffers into its static inputs
                g.meta_stage.copy_(host, non_blocking = True)
                POOL.give(raw)
                lat_bytes = model._latents_into(rb, g.lat_stage)
                staged = torch.cuda.Event()
                staged.record()
            cur = torch.cuda.current_stream()
            cur.wait_event(staged)
            g.meta.copy_(g.meta_stage, non_blocking = True)
            for dst, src in zip(g.lat, g.lat_stage):
                if dst is not None:
                    dst.copy_(src, non_blocking = True)
            g.consumed.record()
        for t, e in enumerate(g.eps):
            if e is not None:
                if noise is not None and noise[t] is not None:
                    e.copy_(noise[t].reshape(e.shape), non_blocking = True)      # injected (deterministic parity runs)
                else:
                    e.normal_()
        if drop:
            eng.dropout_key(dropout_key, out = g.drop_key)
        if getattr(eng, 'opt_step_dev', None) is None:
            eng.opt_step_dev = torch.zeros(1, device = eng.device, dtype = torch.int32)
        eng.opt_step_dev.fill_(eng.opt_step)             # device-resident optimizer step counter (incremented inside the graph)
        if g.graph is None:
            if self.ema_decay is not None and getattr(eng, 'ema_flat', None) is None:
                eng.ema_flat = eng.flat.clone()          # must exist before the capture (an allocation + copy inside it would be replayed)
            import copy
            eng.pin_workspaces()                         # workspace buffers that later have to grow are retired, not freed
            g.rb = copy.copy(rb)                         # descriptor object whose device views point into the static metadata buffer
            g.rb.dev = eng.meta_views(rb, g.meta, layout)
            rb = g.rb
            eng.zero_grad()
            eng._dirty = True                            # the capture must contain the weight repack that follows every optimizer step
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            l0 = eng.ops.launches
            with torch.cuda.graph(graph):
                res = eng.forward(rb, g.lat, g.eps, train = True, text_loss_weight = model.text_loss_weight, flow_loss_weight = model.flow_loss_weight,
                                  dropout = model.training, dropout_key = g.drop_key, recon_weight = model.reconstruction_loss_weight if recon else 0.)
                # NCCL all-reduce of the flat gradient buffer captured INSIDE the step graph: per-layer buckets on the communication stream, forked
                # from / joined to the capture stream, so the collective of layers >= i overlaps the backward kernels of layers < i on every replay
                self._backward_allreduce(eng, lambda cb: eng.backward(bucket_cb = cb))
                if self.max_grad_norm is not None:
                    eng.clip_grad_norm_(self.max_grad_norm, 1.0 / self.world)
                eng.adam_step(grad_scale = 1.0 / self.world, zero_grads = True, device_step = True, **self.hp)
                if self.ema_decay is not None:
                    eng.ema_update(self.ema_decay)
                g.loss = res['total']
            eng.opt_step -= 1                            # the capture itself executed nothing
            g.launches = eng.ops.launches - l0           # kernels of ours inside one replay
            eng.ops.launches = l0
            g.graph = graph
            g.pins = (dict(eng.ws), dict(eng.packed), eng.fastp, eng.flat, eng.gflat, eng.exp_avg, eng.exp_avg_sq)   # every address the graph baked in
        eng.opt_step += 1
        eng._grads_clean = True                          # the graph ends with the Adam pass that clears the gradient buffer
        g.graph.replay()
        eng.ops.launches += g.launches
        eng._dirty = True                                # parameters changed: the bf16 operand copies are repacked at the start of the next step
        model._last_batch = g.rb
        g.rb.dev['h2d_bytes'] = g.meta.numel() * 4
        g.rb.latent_h2d_bytes = lat_bytes
        return g.loss.clone()

    # ---- engine-backed (CUDA) path
    def _bucket_bounds(self, eng):
        """flat-buffer offset where each layer's parameters start (layers are contiguous in named_parameters order)"""
        if getattr(self, '_bounds', None) is None:
            # conditioning-path parameters live in the "late" region of the flat buffer (engine.attach): their gradients are only
            # final after backward() returns, so they are never part of a per-layer bucket
            starts = {}
            for name, off in eng.offs.items():
                if name.startswith('transformer.layers.') and off < eng.late_start:
                    i = int(name.split('.')[2])
                    starts[i] = min(starts.get(i, 1 << 62), off)
            self._bounds = starts
            self._tail = max((off + eng.named[n].numel() for n, off in eng.offs.items() if n.startswith('transformer.layers.') and off < eng.late_start), default = 0)
        return self._bounds

    def _bucket_cb(self, eng):
        """callback for `Engine.backward(bucket_cb=)`: all-reduce the flat-gradient slice of the layers whose backward kernels have just been enqueued,
        on the communication stream, behind an event recorded on the compute stream (works eagerly and under CUDA-graph capture, where the event
        record / wait become fork / join edges of the graph)."""
        bounds = self._bucket_bounds(eng)
        if self.comm_stream is None:
            self.comm_stream = torch.cuda.Stream()
        hi = [self._tail]
        def cb(i):
            lo = bounds[i]
            if (hi[0] - lo) * 4 < self.bucket_bytes and i > 0:
                return                                            # keep growing the bucket (~25 MB buckets: launch latency vs overlap)
            ev = torch.cuda.Event(); ev.record()
            with torch.cuda.stream(self.comm_stream):
                self.comm_stream.wait_event(ev)
                dist.all_reduce(eng.gflat[lo:hi[0]])
            hi[0] = lo
        def finish():
            ev = torch.cuda.Event(); ev.record()
            with torch.cuda.stream(self.comm_stream):
                self.comm_stream.wait_event(ev)
                if hi[0] > 0:
                    dist.all_reduce(eng.gflat[:hi[0]])
                if self._tail < eng.gflat.numel():
                    dist.all_reduce(eng.gflat[self._tail:])   # final norm, heads, embedding and the conditioning ("late") parameters
            torch.cuda.current_stream().wait_stream(self.comm_stream)
        return cb, finish

    def _backward_allreduce(self, eng, run_backward):
        """backward + gradient all-reduce: per-layer buckets overlapped with the rest of backward (`overlap`), or one call afterwards"""
        if self.world > 1 and self.overlap:
            cb, finish = self._bucket_cb(eng)
            run_backward(cb)
            finish()
        else:
            run_backward(None)
            if self.world > 1:
                dist.all_reduce(eng.gflat)

    def step_packed_eager(self, rb, latents, noise = None, dropout_key = None):
        """the step of `step_packed` launched eagerly (profiling passes, shapes that are not captured)"""
        model, eng = self.model, self.model.engine
        eng.ensure_attached()
        self._sync_replicas(eng)
        eng.upload(rb)
        eng.zero_grad()
        loss = model.forward_packed(rb, latents, noise = noise, dropout_key = dropout_key)
        def run(cb):
            eng._bucket_cb = cb
            loss.backward()
            eng._bucket_cb = None
        self._backward_allreduce(eng, run)
        self._finish_step(eng)
        return loss

    def _finish_step(self, eng):
        """[clip] -> fused Adam (clears the gradient buffer: the next step's zero_grad() is free) -> [EMA]"""
        if self.max_grad_norm is not None:
            eng.clip_grad_norm_(self.max_grad_norm, 1.0 / self.world)
        eng.adam_step(grad_scale = 1.0 / self.world, zero_grads = True, **self.hp)
        if self.ema_decay is not None:
            eng.ema_update(self.ema_decay)

    def step_packed(self, rb, latents, noise = None, dropout_key = None):
        """One training step from a packed batch that is already resident on the device (`model.pack` + `engine.upload` + latents on the
        device): CUDA-graph replay when the shape signature has been seen before, eager launches otherwise.  Single process only.
        `noise` / `dropout_key` (optional): injected flow noise and dropout key (`Transfusion.forward`) for deterministic runs."""
        model, eng = self.model, self.model.engine
        eng.ensure_attached()
        self._sync_replicas(eng)
        eng.upload(rb)
        loss = self._graph_step(rb, device_lat = latents, noise = noise, dropout_key = dropout_key) if self.cuda_graph else None
        if loss is None:
            loss = self.step_packed_eager(rb, latents, noise = noise, dropout_key = dropout_key)
        return loss

    def step(self, batch, times = None, noise = None, **fw):
        """`noise` (optional, per modality type `[S_t, dim_latent]`): injected flow noise for deterministic parity runs"""
        model = self.model
        eng = model.engine
        cuda = hasattr(eng, 'gflat') or model.device.type == 'cuda'
        if cuda:
            eng.ensure_attached()
            self._sync_replicas(eng)
            if self.cuda_graph and model.training and not fw and torch.is_grad_enabled():
                rb, _ = model.pack(batch, times = times)
                dnoise = [n.reshape(-1, model.dim_latents[t]).float().to(model.device) if n is not None else None for t, n in enumerate(noise)] if noise is not None else None
                loss = self._graph_step(rb, noise = dnoise)
                if loss is not None:
                    return loss
                eng.zero_grad()
                loss = model.forward_packed(rb, model._latents_to_device(rb), noise = dnoise)
            else:
                eng.zero_grad()
                loss = model(batch, times = times, noise = noise, **fw)
        else:
            for p in model.parameters():
                p.grad = None
            loss = model(batch, times = times, noise = noise, **fw)
        # Eager and captured steps issue the SAME sequence of collectives (same bucket boundaries), so ranks whose batches have different shape
        # signatures (one replaying a graph, one still launching eagerly) stay in lock-step on the communicator.
        if cuda:
            def run(cb):
                eng._bucket_cb = cb
                loss.backward()
                eng._bucket_cb = None
            self._backward_allreduce(eng, run)
        else:
            loss.backward()
            if self.world > 1:
                grads = [p.grad for p in model.parameters() if p.grad is not None]
                flat = torch._utils._flatten_dense_tensors(grads)
                dist.all_reduce(flat)
                for g, f in zip(grads, torch._utils._unflatten_dense_tensors(flat, grads)):
                    g.copy_(f)
        if cuda:
            self._finish_step(eng)
        else:
            if self._cpu_opt is None:
                cls = torch.optim.AdamW if self.hp['decoupled'] else torch.optim.Adam
                self._cpu_opt = cls(model.parameters(), lr = self.hp['lr'], betas = self.hp['betas'], eps = self.hp['eps'], weight_decay = self.hp['weight_decay'])
            if self.world > 1:
                for p in model.parameters():
                    if p.grad is not None:
                        p.grad.div_(self.world)
            if self.max_grad_norm is not None:
                torch.nn.utils.clip_grad_norm_(list(model.parameters()), self.max_grad_norm)
            self._cpu_opt.step()
        return loss
