"""CUDA-graph replay and encoder/search pipelining of a planner's inference forward for fixed batch shapes.

An eager `planner(map_designs, start_maps, goal_maps)` issues half a dozen launches from Python (first layer /
pack kernel, encoder convs, head kernel, search kernel); at 32x32 / batch 100 the GPU work is ~0.4 ms on an H100, so
the step is close to CPU-launch bound and slows down further when several ranks share a host (SURVEY.md 8(f) rank 3).

    fast = GraphedPlanner(planner, map_designs, start_maps, goal_maps)   # example batch fixes shapes/dtypes
    out = fast(map_designs, start_maps, goal_maps)                        # AstarOutput, caller-owned tensors
    out = fast.replay_host()      # inputs read from fast.host_inputs (pinned), outputs land in fast.host_outputs:
                                  # H2D copies, forward and D2H copies are ONE graph launch

    pipe = PipelinedPlanner(planner, map_designs, start_maps, goal_maps)
    for batch in batches:                      # search(k) overlaps encoder(k+1) inside one graph launch per step
        prev = pipe.submit(*batch)             # AstarOutput of the PREVIOUS batch (None for the first)
    last = pipe.drain()

    over = OverlappedPlanner(planner, n_streams=4)     # any planner, any shapes: consecutive batches on several streams
    handles = [over.submit(*batch) for batch in batches]
    outs = [h.result() for h in handles]               # each result() orders the current stream after that batch

Inference only (eval mode, no autograd, `store_intermediate_results=False`).  Batches of more than one map with
`g_ratio < 0.5` are searched batch-coupled, as the eager call does; inside the graphs T_batch is decided on the device
(`_native.forward_coupled`) instead of by the eager call's host round trip, with the same outputs.
"""
from __future__ import annotations

from typing import Optional

import torch

from ..planner.differentiable_astar import AstarOutput


def _check_planner(planner, map_designs):
    if planner.training:
        raise ValueError("graph capture covers the inference forward: call planner.eval() first")
    dev = next((p.device for p in planner.parameters()), torch.device("cuda", torch.cuda.current_device()))
    if dev.type != "cuda":
        raise ValueError("the planner must live on a CUDA device")
    return dev


def _warm(planner, inputs, dev, warmup):
    """cuDNN autotuning, plan building (one host sync) and lazy one-time initialisation, outside capture."""
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side), torch.no_grad():
        for _ in range(max(1, warmup)):
            planner(*inputs)
    torch.cuda.current_stream(dev).wait_stream(side)
    torch.cuda.synchronize(dev)


class GraphedPlanner:
    def __init__(self, planner: torch.nn.Module, map_designs: torch.Tensor, start_maps: torch.Tensor,
                 goal_maps: torch.Tensor, device=None, warmup: int = 3):
        dev = _check_planner(planner, map_designs) if device is None else torch.device(device)
        self.planner = planner
        self.device = dev
        examples = (map_designs, start_maps, goal_maps)
        self._in = tuple(torch.empty(t.shape, dtype=t.dtype, device=dev) for t in examples)
        for dst, src in zip(self._in, examples):
            dst.copy_(src)
        _warm(planner, self._in, dev, warmup)
        from .. import _native

        before = _native.launch_count()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph), torch.no_grad():
            out = planner(*self._in)
        self._out = out
        # kernels of libnastar_b200 recorded in the graph: each replay launches them again without going through
        # the library's host entry points (so nastar_b200_launch_count() does not see replays)
        self.native_launches_per_replay = _native.launch_count() - before
        self.replays = 0
        # end-to-end variant: pinned host buffers -> device -> forward -> pinned host buffers, one graph
        self._host_in = tuple(torch.empty(t.shape, dtype=t.dtype).pin_memory() for t in examples)
        for dst, src in zip(self._host_in, examples):
            dst.copy_(src)
        self._host_out = (torch.empty(out.histories.shape, dtype=out.histories.dtype).pin_memory(),
                          torch.empty(out.paths.shape, dtype=out.paths.dtype).pin_memory())
        self._graph_host: Optional[torch.cuda.CUDAGraph] = None
        self._out_host: Optional[AstarOutput] = None

    @property
    def static_inputs(self):
        """(map_designs, start_maps, goal_maps) buffers the graph reads; fill them and call replay() to skip copies."""
        return self._in

    @property
    def static_outputs(self) -> AstarOutput:
        """Outputs of the last replay, owned by the graph (overwritten by the next replay)."""
        return self._out

    @property
    def host_inputs(self):
        """Pinned host staging buffers read by replay_host() (write the next batch here)."""
        return self._host_in

    @property
    def host_outputs(self):
        """(histories, paths) pinned host buffers written by replay_host(); valid after a stream/event sync."""
        return self._host_out

    def replay(self) -> AstarOutput:
        self.graph.replay()
        self.replays += 1
        return self._out

    def replay_host(self) -> AstarOutput:
        """One graph launch: H2D of host_inputs, the forward, D2H into host_outputs.  Returns the device-side
        outputs (graph-owned); the host copies complete in stream order."""
        if self._graph_host is None:
            torch.cuda.synchronize(self.device)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g), torch.no_grad():
                ins = tuple(torch.empty_like(d) for d in self._in)
                for d, h in zip(ins, self._host_in):
                    d.copy_(h, non_blocking=True)
                out = self.planner(*ins)
                self._host_out[0].copy_(out.histories, non_blocking=True)
                self._host_out[1].copy_(out.paths, non_blocking=True)
            self._graph_host, self._out_host = g, out
        self._graph_host.replay()
        self.replays += 1
        return self._out_host

    def __call__(self, map_designs: torch.Tensor, start_maps: torch.Tensor, goal_maps: torch.Tensor,
                 store_intermediate_results: bool = False) -> AstarOutput:
        if store_intermediate_results:
            raise ValueError("store_intermediate_results needs a host sync per call; use the eager planner")
        for dst, src in zip(self._in, (map_designs, start_maps, goal_maps)):
            if src.shape != dst.shape or src.dtype != dst.dtype:
                raise ValueError(f"GraphedPlanner was captured for {tuple(dst.shape)} {dst.dtype}, got {tuple(src.shape)} {src.dtype}")
            dst.copy_(src, non_blocking=True)
        self.graph.replay()
        self.replays += 1
        return AstarOutput(self._out.histories.clone(), self._out.paths.clone(), [])


class _Pending:
    """Outputs of one OverlappedPlanner.submit(): valid for the caller's stream after result()."""

    def __init__(self, output: AstarOutput, event: torch.cuda.Event, stream: torch.cuda.Stream):
        self._output, self._event, self._stream = output, event, stream

    def done(self) -> bool:
        return self._event.query()

    def result(self) -> AstarOutput:
        """Make the current stream wait for this batch (no host block) and hand the outputs over to it."""
        cur = torch.cuda.current_stream(self._output.histories.device)
        cur.wait_event(self._event)
        for t in (self._output.histories, self._output.paths):
            t.record_stream(cur)
        return self._output


class OverlappedPlanner:
    """Throughput mode for searches with a long tail: consecutive batches go round-robin onto `n_streams` streams.

    A search launch lasts as long as its longest map while most SMs have run out of work long before (Config 5,
    1024 random 256x256 maps: mean 507 steps, longest 12 616 — 7.3 ms per launch, 141 k maps/s on one H100 SXM at
    700 W).  The large-map engines run persistent CTAs that exit as their work queue drains, so a launch enqueued on
    ANOTHER stream moves onto the vacated SMs while the previous batch's long maps finish on a few: 2.89 ms per batch
    = 354 k maps/s on the same H100 with 4 streams.  Works with any planner and any shapes (plain eager calls, no
    graph capture); each batch's results are identical to a direct call.  Inputs must stay unmodified until the batch has run (they are read
    asynchronously); outputs are owned by the caller after result().
    """

    def __init__(self, planner: torch.nn.Module, n_streams: int = 4, device=None):
        if n_streams < 1:
            raise ValueError("n_streams must be >= 1")
        dev = device if device is not None else next((p.device for p in planner.parameters()),
                                                     torch.device("cuda", torch.cuda.current_device()))
        dev = torch.device(dev)
        if dev.type != "cuda":
            raise ValueError("OverlappedPlanner needs a CUDA device")
        self.planner, self.device = planner, dev
        self._streams = [torch.cuda.Stream(device=dev) for _ in range(n_streams)]
        self._k = 0

    def submit(self, map_designs: torch.Tensor, start_maps: torch.Tensor, goal_maps: torch.Tensor) -> _Pending:
        st = self._streams[self._k % len(self._streams)]
        self._k += 1
        st.wait_stream(torch.cuda.current_stream(self.device))     # the inputs were produced on the caller's stream
        with torch.cuda.stream(st), torch.no_grad():
            for t in (map_designs, start_maps, goal_maps):
                t.record_stream(st)
            out = self.planner(map_designs, start_maps, goal_maps)
            ev = torch.cuda.Event()
            ev.record(st)
        return _Pending(out, ev, st)

    def wait_all(self) -> None:
        """Order the current stream after everything submitted so far (outputs stay with their handles)."""
        cur = torch.cuda.current_stream(self.device)
        for st in self._streams:
            cur.wait_stream(st)


class PipelinedPlanner:
    """Software pipeline over consecutive batches of a NeuralAstar: while the search kernel of batch k runs on a
    hundred warps, the encoder convolutions of batch k+1 occupy the tensor cores.  Both are branches of one CUDA
    graph (captured with forked streams), multi-buffered on inputs, encoder output and results; a step is ONE
    graph launch.  Outputs are identical to the eager call's (same kernels, same order per batch).

    Device inputs (default): two stages.  submit(batch k) runs  encoder(k) || search(k-1)  and returns the outputs of
    batch k-1.

    `host=True` builds the end-to-end variant, three stages deep: submit() number k runs
        H2D(batch k, from the pinned `host_inputs[k % 3]`)  ||  encoder(k-1)  ||  search(k-2) -> D2H into the pinned
        `host_outputs[k % 2]`
    so both PCIe copies (1.2 MB each way per batch of 100 32x32 maps) hide behind the convolutions.  Batch k's results
    are complete once submit() number k+2 (or drain()) has finished.

    `fork` places the search inside the step: "late" right before the encoder's last, widest convolution (the default
    of the device pipeline), "early" at the start of the step (the default of host=True).  Late puts the search
    beside the fused conv4 + head kernel, whose CTAs leave room for one search warp on every SM sub-partition.  Measured on an H100 80GB HBM3 at a 700 W power limit
    (tools/pipe_breakdown.py, b=100, 32x32): the encoder branch alone takes 281 us and the search branch 76 us; the
    device step takes 298 us forked late and 306 us forked early, the three-stage host step 314 us late and 305 us
    early.  Before the fused kernel left that room, late cost 360 us against 314 us early on the same card.
    """

    def __init__(self, planner: torch.nn.Module, map_designs: torch.Tensor, start_maps: torch.Tensor,
                 goal_maps: torch.Tensor, host: bool = False, warmup: int = 3, fork: Optional[str] = None):
        from ..planner.astar import NeuralAstar

        if not isinstance(planner, NeuralAstar):
            raise TypeError("PipelinedPlanner overlaps an encoder with the search: it needs a NeuralAstar")
        dev = _check_planner(planner, map_designs)
        if fork is None:
            fork = "early" if host else "late"
        if fork not in ("late", "early"):
            raise ValueError("fork must be 'late' or 'early'")
        self.planner, self.device, self.host, self.fork = planner, dev, host, fork
        examples = (map_designs, start_maps, goal_maps)
        n_in = 3 if host else 2      # input buffers: H2D(k) || encoder(k-1) || search(k-2) touch three different batches
        # when the three inputs share shape and dtype (the "m+" planners) they live in ONE stacked buffer per
        # slot, so a whole batch can arrive with a single copy (submit_stacked)
        self._stacked = None
        if all(t.shape == map_designs.shape and t.dtype == map_designs.dtype for t in examples):
            self._stacked = [torch.empty((3,) + tuple(map_designs.shape), dtype=map_designs.dtype, device=dev)
                             for _ in range(n_in)]
            self._in = [tuple(st[i] for i in range(3)) for st in self._stacked]
        else:
            self._in = [tuple(torch.empty(t.shape, dtype=t.dtype, device=dev) for t in examples) for _ in range(n_in)]
        for buf in self._in:
            for dst, src in zip(buf, examples):
                dst.copy_(src)
        _warm(planner, self._in[0], dev, warmup)
        with torch.no_grad():
            head = self._encode(self._in[0])
        if head is None:
            raise ValueError("this planner/shape has no fused encoder hand-off (needs a conv head and a grid <= 64x64)")
        taps, self._bias, self._scale = head
        self._taps = [torch.empty_like(taps) for _ in range(2)]
        self._host_in = self._host_out = None
        if host:
            self._host_in = [tuple(torch.empty(t.shape, dtype=t.dtype).pin_memory() for t in examples) for _ in range(n_in)]
            for buf in self._host_in:
                for dst, src in zip(buf, examples):
                    dst.copy_(src)
            B, _, H, W = start_maps.shape
            self._host_out = [(torch.empty((B, 1, H, W), dtype=torch.float32).pin_memory(),
                               torch.empty((B, 1, H, W), dtype=torch.int64).pin_memory()) for _ in range(2)]
        self._side = torch.cuda.Stream(device=dev)
        self._copy = torch.cuda.Stream(device=dev) if host else None
        self._graphs = {}
        self._outs = {}
        self._k = 0            # batches submitted so far
        self.replays = 0
        from .. import _native

        self._native = _native
        self.native_launches = 0   # library kernels launched by graph replays (not seen by launch_count())
        self._per_graph = {}

    # -- building blocks ---------------------------------------------------------------------------------
    def _encode(self, ins, out=None, on_last_conv=None):
        p = self.planner
        return p._head_taps(*ins, out=out, on_last_conv=on_last_conv)

    def _search(self, in_idx: int, taps_idx: int):
        p = self.planner
        ins = self._in[in_idx]
        passable = torch.ones_like(ins[1]) if p.learn_obstacles else ins[0]
        return p.astar.search_from_taps(self._taps[taps_idx], self._bias, self._scale, ins[1], ins[2], passable)

    def _step_graph(self, k: int, copy: bool, enc: bool, search: bool):
        """One step as a graph.  Host pipeline: `copy` = H2D of batch k, `enc` = encoder of batch k-1, `search` = search
        (+ D2H) of batch k-2.  Device pipeline (no copy stage): `enc` = encoder of batch k, `search` = search of batch
        k-1.  Buffer slots depend on k only through k mod 6 (inputs cycle mod 3 or 2, encoder outputs mod 2)."""
        lag = 1 if self.host else 0
        n_in = len(self._in)
        key = (k % (6 if self.host else 2), copy, enc, search)
        if key in self._graphs:
            return key
        e, s_ = k - lag, k - lag - 1           # batch numbers of the encoder / search stage
        torch.cuda.synchronize(self.device)
        before = self._native.launch_count()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g), torch.no_grad():
            main = torch.cuda.current_stream(self.device)
            forked = []

            def fork_search():
                if forked:
                    return
                self._side.wait_stream(main)                       # fork
                with torch.cuda.stream(self._side):
                    res = self._search(s_ % n_in, s_ % 2)
                    if self.host:
                        self._host_out[s_ % 2][0].copy_(res.histories, non_blocking=True)
                        self._host_out[s_ % 2][1].copy_(res.paths, non_blocking=True)
                forked.append(res)

            if copy:
                self._copy.wait_stream(main)                       # fork
                with torch.cuda.stream(self._copy):
                    for d, h in zip(self._in[k % n_in], self._host_in[k % n_in]):
                        d.copy_(h, non_blocking=True)
            if search and (self.fork == "early" or not enc):
                fork_search()
            if enc:
                self._encode(self._in[e % n_in], out=self._taps[e % 2], on_last_conv=fork_search if search else None)
            if search:
                fork_search()                                      # encoders that never reached the hook
                main.wait_stream(self._side)                       # join
            if copy:
                main.wait_stream(self._copy)                       # join
        self._graphs[key] = g
        self._outs[key] = forked[0] if forked else None
        self._per_graph[key] = self._native.launch_count() - before
        return key

    def _run(self, key):
        self._graphs[key].replay()
        self.replays += 1
        self.native_launches += self._per_graph[key]
        return self._outs[key]

    # -- public API --------------------------------------------------------------------------------------
    @property
    def depth(self) -> int:
        """Stages between submit(batch k) and its results: 2 (device inputs) or 3 (host=True)."""
        return 3 if self.host else 2

    @property
    def host_inputs(self):
        """[(map_designs, start_maps, goal_maps)] x 3 pinned staging buffers; batch k is read from index k % 3."""
        return self._host_in

    @property
    def host_outputs(self):
        """[(histories, paths)] x 2 pinned result buffers; batch k lands in index k % 2 during submit() number k+2
        (or drain())."""
        return self._host_out

    def submit(self, map_designs: Optional[torch.Tensor] = None, start_maps: Optional[torch.Tensor] = None,
               goal_maps: Optional[torch.Tensor] = None) -> Optional[AstarOutput]:
        """Enqueue batch k.  Device pipeline: pass the three device tensors; returns the graph-owned outputs of batch
        k-1 (overwritten two submits later), None for the first batch.  host=True: pass nothing, the batch is read
        from host_inputs[k % 3]; returns the device outputs of batch k-2 (None for the first two) whose copies are
        landing in host_outputs[k % 2]."""
        k = self._k
        if self.host:
            key = self._step_graph(k, True, k >= 1, k >= 2)
        else:
            for dst, src in zip(self._in[k & 1], (map_designs, start_maps, goal_maps)):
                dst.copy_(src, non_blocking=True)
            key = self._step_graph(k, False, True, k >= 1)
        self._k += 1
        return self._run(key)

    def submit_stacked(self, batch: torch.Tensor) -> Optional[AstarOutput]:
        """submit() for a batch delivered as one [3, B, 1, H, W] tensor (map_designs, start_maps, goal_maps stacked):
        a single device copy instead of three."""
        if self._stacked is None or self.host:
            raise ValueError("submit_stacked needs equally shaped inputs and a device-input pipeline")
        k = self._k
        self._stacked[k & 1].copy_(batch, non_blocking=True)
        key = self._step_graph(k, False, True, k >= 1)
        self._k += 1
        return self._run(key)

    def drain(self) -> Optional[AstarOutput]:
        """Finish every submitted batch; returns the outputs of the last one.  The pipeline is empty afterwards."""
        k = self._k
        if k == 0:
            return None
        out = None
        if self.host:
            out = self._run(self._step_graph(k, False, True, k >= 2))         # encoder(k-1) || search(k-2)
            out = self._run(self._step_graph(k + 1, False, False, True))      # search(k-1)
        else:
            out = self._run(self._step_graph(k, False, False, True))          # search(k-1)
        self._k = 0
        return out

    def prepare(self) -> None:
        """Capture every graph variant now (otherwise captured lazily on first use, which synchronises)."""
        if self.host:
            self._step_graph(0, True, False, False)
            self._step_graph(1, True, True, False)
            self._step_graph(1, False, True, False)                          # drain after a single batch
            for k in range(2, 8):
                self._step_graph(k, True, True, True)
                self._step_graph(k, False, True, True)
                self._step_graph(k, False, False, True)
        else:
            self._step_graph(0, False, True, False)
            for k in (1, 2):
                self._step_graph(k, False, True, True)
                self._step_graph(k, False, False, True)
