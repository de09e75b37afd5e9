"""Incremental decoding state of the causal Hyena operator (the reference leaves HyenaOperator.recurrence unimplemented,
src/models/sequence/hyena.py:384-386, and ignores the ``inference_params`` that LMBackbone threads through,
src/models/sequence/long_conv_lm.py:375-376).

Output t of the causal recurrence o (hyena.py:414-423) is
    out_o[t] = sum_{s<=t} k_o[t-s] g_o[s] + bias_o g_o[t],    g_o = v_o * x_{O-1-o},
so extending a sequence by one position needs the gated inputs g_o of every earlier position, the filter k and the last
two in_proj outputs (the state of the 3-tap short filter) -- not a forward over the whole sequence.  ``DecodeCache`` holds
exactly that; ``HyenaOperator.prefill`` / ``step`` fill and use it (csrc/decode.cuh).

The filter is generated once, at allocation, for Lcap = min(max_seqlen, l_max) positions.  That is valid for any shorter
prefix: k[j] depends on position j only -- z and t are sliced per position, the modulation is per position and the
``normalized`` option divides by the L1 norm over channels at each position (hyena.py:235-236).
"""
import torch

from ._lib import HyenaB200Error

CHUNK = 1024          # positions per partial dot product of a step (csrc/decode_args.h kChunk)


def _ld(lcap):
    return (lcap + 3) // 4 * 4


def _chunks(lcap):
    return (lcap + CHUNK - 1) // CHUNK


def _host_index(index, n, what):
    """index (a sequence or 1-D tensor of integers) -> list of ints in [0, n), checked on the host before any device work."""
    if torch.is_tensor(index):
        if index.dim() != 1 or index.dtype.is_floating_point or index.dtype.is_complex or index.dtype == torch.bool:
            raise HyenaB200Error(f"{what} must be a 1-D integer index; got {index.dtype} of shape {tuple(index.shape)}")
        index = index.tolist()
    try:
        out = [int(i) for i in index]
        if any(isinstance(i, bool) or int(i) != i for i in index):
            raise ValueError
    except (TypeError, ValueError):
        raise HyenaB200Error(f"{what} must be a 1-D sequence of integers") from None
    if not out:
        raise HyenaB200Error(f"{what} is empty")
    bad = [i for i in out if not 0 <= i < n]
    if bad:
        raise HyenaB200Error(f"{what} {bad[0]} outside [0, {n})")
    return out


class _PositionState:
    """The values last written to a device position (None: unknown), shared by every cache that holds the tensor."""

    def __init__(self):
        self.value = None


class DecodeCache:
    """Decoding state of one HyenaOperator (``HyenaOperator.allocate_decode_cache``), or of every mixer of a stack
    (``Backbone.allocate_decode_cache``: ``layers`` holds one per layer, looked up by module identity).

    Per operator, with O = order, D = d_model, F = (O-1) D filter channels, C = (O+1) D in_proj channels and ld = Lcap
    rounded up to a multiple of 4 (all fp32, on the operator's device):
      k     (F * ld + 4,)       the filter, each row time-reversed (k[c][j] at c*ld + ld-1-j) so that the step kernel streams
                                history and filter in ascending order; 4 floats of padding
      bias  (F,)                the effective filter bias (0 * bias when use_bias is false, as in forward)
      h     (O-1, B, D, ld)     g_o of every recurrence by position
      tail  (B, C, 2)           in_proj outputs (with bias) of the last two positions
      s_t   (B, C)              short-filter outputs of the current position
      part  (B, D, ceil(Lcap / 1024))  partial dot products of one step
    ``t`` is the number of positions consumed so far.

    Window state of the windowed step (ops.decode_window_plan, DESIGN.md section 4.11): a window [win_b, win_b + win_wc)
    is valid while win_b <= t < win_b + win_wc; ``win_f`` (O-1, B, D, W) holds F_o[j] = sum_{s < win_b} k_o[win_b+j-s]
    g_o[s] for j < win_wc.  F depends on h[:, :, :, :win_b] only, so an extend inside the window leaves it valid.  It is
    allocated at the first refresh (``window_nbytes``).  ``steps`` counts the steps since the last prefill or extend.

    A *branched* cache (``fork``, ``select``; DESIGN.md section 4.12) holds R branches that continue rows of a parent cache
    from its position t0.  With base b = t0 - t0 mod 4, Hc = min(horizon rounded up to a multiple of 4, Lcap - b) and
    H = Hc rounded up to a multiple of 4, per operator:
      k, bias                the parent's (shared: never written after allocation)
      h     (O-1, R, D, H)   g_o of each branch at positions [b, b + Hc)
      f     (O-1, P, D, H)   F_o[p][j] = sum_{s<b} k_o[b+j-s] g_o[s] of the P distinct forked parent rows, j < Hc
      parent (R,) int32      the row of f each branch reads
      tail, s_t, part        as above with R rows and ceil(H / 1024) partials
    so out_o[t] = F_o[parent][t-b] + sum_{b<=s<t} k_o[t-s] g_o[s] + (k_o[0] + bias_o) g_o[t] for b <= t < b + Hc, and no
    operation on a branch reads the context before b.

    Device position (``sync_position``, StepGraph): ``pos`` (3,) int32 on the device holds [t, win_b, base] for the step
    kernels that read the position on the device.  One tensor serves every layer of a stack.  It is allocated on first
    use and written only by ``sync_position`` and by a replayed StepGraph; ``t`` on the host stays authoritative."""

    def __init__(self, owner=None, batch_size=0, max_seqlen=0, lcap=0, k=None, bias=None, h=None, tail=None, s_t=None,
                 part=None, layers=None):
        self.owner = owner
        self.batch_size, self.max_seqlen, self.lcap = int(batch_size), int(max_seqlen), int(lcap)
        self.k, self.bias, self.h, self.tail, self.s_t, self.part = k, bias, h, tail, s_t, part
        self.layers = list(layers) if layers is not None else []
        self._t = 0
        self.win_b, self.win_wc, self.win_f, self.steps = 0, 0, None, 0
        self._branched, self.base, self.hc, self.f, self.parent = False, 0, 0, None, None
        self.pos, self._pos_state = None, None
        if owner is not None:
            self.d_model, self.order = owner.d_model, owner.order

    @classmethod
    def allocate(cls, op, batch_size, max_seqlen):
        """Decoding state of ``op`` for ``batch_size`` rows and up to min(max_seqlen, op.l_max) positions."""
        if op.filter_fn.bidirectional:
            raise HyenaB200Error("decoding needs a causal filter; this HyenaFilter is bidirectional")
        if batch_size < 1 or max_seqlen < 1:
            raise HyenaB200Error(f"allocate_decode_cache: batch_size {batch_size} and max_seqlen {max_seqlen} must be >= 1")
        w = op.in_proj.weight
        if not w.is_cuda:
            raise HyenaB200Error("decoding runs on CUDA sm_90a only; the operator's parameters are on the CPU")
        B, D, O = int(batch_size), op.d_model, op.order
        lcap = min(int(max_seqlen), op.l_max)
        ld = _ld(lcap)
        F = (O - 1) * D
        dev = w.device
        with torch.no_grad():
            k = op.filter_fn.filter_channel_major(lcap)                  # (F, lcap)
            krev = torch.zeros(F * ld + 4, dtype=torch.float32, device=dev)
            krev[:F * ld].view(F, ld)[:, ld - lcap:] = k.flip(-1)
            fb = op.filter_fn.bias if op.filter_fn.use_bias else 0 * op.filter_fn.bias
            fb = fb.detach().reshape(-1).to(torch.float32).contiguous().clone()
        h = torch.zeros(O - 1, B, D, ld, dtype=torch.float32, device=dev)
        tail = torch.zeros(B, (O + 1) * D, 2, dtype=torch.float32, device=dev)
        s_t = torch.zeros(B, (O + 1) * D, dtype=torch.float32, device=dev)
        part = torch.zeros(B, D, _chunks(lcap), dtype=torch.float32, device=dev)
        return cls(op, B, max_seqlen, lcap, krev, fb, h, tail, s_t, part)

    @classmethod
    def stack(cls, caches):
        """One cache for several operators (one per layer of a stack), each found by ``for_module``."""
        caches = list(caches)
        if not caches:
            raise HyenaB200Error("DecodeCache.stack needs at least one operator cache")
        return cls(None, caches[0].batch_size, caches[0].max_seqlen, min(c.lcap for c in caches), layers=caches)

    @staticmethod
    def layout_nbytes(batch_size, d_model, order, lcap):
        """Bytes one operator's cache takes (the layout in the class docstring)."""
        B, D, O = batch_size, d_model, order
        ld, F, C = _ld(lcap), (order - 1) * d_model, (order + 1) * d_model
        return 4 * ((F * ld + 4) + F + (O - 1) * B * D * ld + B * C * 2 + B * C + B * D * _chunks(lcap))

    @property
    def nbytes(self):
        """Bytes the cache owns: the layout above, or for a branched cache its branch state (h, f, tail, s_t, part, parent;
        the filter is the parent's)."""
        if self.layers:
            return sum(c.nbytes for c in self.layers)
        own = (self.h, self.f, self.tail, self.s_t, self.part, self.parent) if self.branched else \
              (self.k, self.bias, self.h, self.tail, self.s_t, self.part)
        return sum(x.numel() * x.element_size() for x in own)

    @property
    def branched(self):
        return self.layers[0].branched if self.layers else self._branched

    def fork(self, rows, horizon=4096):
        """A branched cache of len(rows) rows: row i continues row ``rows[i]`` of this cache from its current position t0
        (repeat a row for several branches of one context) and can be stepped and extended up to horizon positions past
        its base t0 - t0 mod 4, or to Lcap.  A snapshot: this cache can go on decoding without changing the branches.  A
        stack's cache forks every layer."""
        if self.branched:
            raise HyenaB200Error("fork: this cache is branched already; use select() to reorder, repeat or drop branches")
        rows = _host_index(rows, self.batch_size, "fork: rows")
        horizon = int(horizon)
        if horizon < 1:
            raise HyenaB200Error(f"fork: horizon {horizon} must be >= 1")
        for c in (self.layers or [self]):
            if c.owner.filter_fn.bidirectional:
                raise HyenaB200Error("decoding needs a causal filter; this HyenaFilter is bidirectional")
            if c.t < 1 or c.t >= c.lcap:
                raise HyenaB200Error(f"fork: the cache is at position {c.t}; forking needs 1 <= t0 < Lcap = {c.lcap}")
        from . import ops
        if self.layers:
            return DecodeCache.stack(ops.decode_fork(c, rows, horizon) for c in self.layers)
        return ops.decode_fork(self, rows, horizon)

    def select(self, index):
        """A branched cache of the branches ``index`` of this one (repeats allowed): each row copies that branch's history,
        tail and parent row; F is shared.  Reorders, prunes or re-forks beams in one call."""
        if not self.branched:
            raise HyenaB200Error("select: this cache is not branched (fork() first)")
        index = _host_index(index, self.batch_size, "select: index")
        from . import ops
        if self.layers:
            return DecodeCache.stack(ops.decode_select(c, index) for c in self.layers)
        return ops.decode_select(self, index)

    @property
    def window_nbytes(self):
        """Bytes of the windowed step's history tails (0 until the first window opens); not part of ``nbytes``."""
        if self.layers:
            return sum(c.window_nbytes for c in self.layers)
        return 0 if self.win_f is None else self.win_f.numel() * self.win_f.element_size()

    def reset_window(self):
        """Close the window and restart the step count (a prefill starts a new sequence)."""
        self.win_b, self.win_wc, self.steps = 0, 0, 0

    @property
    def t(self):
        return self.layers[0].t if self.layers else self._t

    @t.setter
    def t(self, value):
        if self.layers:
            raise HyenaB200Error("the position of a stack's cache is advanced by its layers")
        self._t = int(value)

    def sync_position(self):
        """The device position ``pos`` = [t, win_b, base] (allocated on first use, one tensor for a stack and all its layers),
        written from the host fields when they differ from the values it was last given."""
        cs = self.layers or [self]
        want = {(c.t, c.win_b, c.base) for c in cs}
        if len(want) != 1:
            raise HyenaB200Error(f"the layers of this stack's cache disagree on (t, win_b, base): {sorted(want)}")
        want = want.pop()
        if self.pos is None or self._pos_state is None:
            pos, state = torch.zeros(3, dtype=torch.int32, device=cs[0].h.device), _PositionState()
            for c in [self] + self.layers:
                c.pos, c._pos_state = pos, state
        if self._pos_state.value != want:
            self.pos.copy_(torch.tensor(want, dtype=torch.int32))
            self._pos_state.value = want
        return self.pos

    def for_module(self, module):
        """The state of ``module`` (this cache itself, or the layer cache allocated for it)."""
        if self.owner is module:
            return self
        for c in self.layers:
            if c.owner is module:
                return c
        raise HyenaB200Error("this DecodeCache was not allocated for this HyenaOperator")


class StepGraph:
    """``step`` of a HyenaOperator, Block or Backbone on one cache, captured in CUDA graphs and replayed per position.

    An eager step costs about 0.1 ms of host and launch time per operator (DESIGN.md section 4.13).  Here the whole step --
    the projections, the step kernels, the add + LayerNorm kernels, the block MLP and ln_f -- is one graph launch.  Its
    kernels read the position from the cache's device position (``DecodeCache.sync_position``), and the last kernel of the
    graph advances it, so every replay steps the next position.  The outputs are the bits eager ``step`` gives on the same
    route.  The routes differ in one case: at t >= WINDOW_MIN_T less than WINDOW_AFTER_STEPS steps after a prefill or an
    extend, eager ``step`` stays on the plain route while a graph step opens a window, whose sums run in another order.

    Routes: the plain step (below ops.WINDOW_MIN_T), the windowed step and the branch step (a branched cache) are separate
    graphs, each captured on first use: warm-up steps on a side stream (their writes to the cache undone), then the capture.
    Before each replay the host runs the route rule on its copy of the position.  When the next position needs a window
    and none holds it, the window is refreshed eagerly, outside the graph, on the current stream: the first step at
    t >= WINDOW_MIN_T opens one, with no run of plain steps before it.  After each replay the host advances ``t`` of every
    layer cache (and the step count of an unbranched one), so eager ``step``, ``extend``, ``fork`` and ``select`` go on
    from there; steps taken eagerly in between are picked up at the next replay.

    ``step`` returns static output tensors that the next ``step`` of this object overwrites: copy what you keep.  It
    raises before any device work on an input of another shape, dtype or device than the captured one, at Lcap or a
    branch horizon, and when a buffer the graphs read was replaced since their capture."""

    WARMUP = 2

    def __init__(self, module, cache, batch_size=None, dtype=torch.float32, residual=False):
        from .block import Backbone, Block
        from .hyena import HyenaOperator
        if isinstance(module, HyenaOperator):
            mixers = [module]
        elif isinstance(module, Block):
            mixers = [module.mixer]
        elif isinstance(module, Backbone):
            mixers = [layer.mixer for layer in module.layers]
        else:
            raise HyenaB200Error(f"StepGraph: expected a HyenaOperator, Block or Backbone; got {type(module).__name__}")
        if not all(isinstance(m, HyenaOperator) for m in mixers):
            raise HyenaB200Error("StepGraph: every mixer must be a HyenaOperator (incremental decoding)")
        if not isinstance(cache, DecodeCache):
            raise HyenaB200Error(f"StepGraph needs a DecodeCache, got {type(cache).__name__}")
        if residual and not isinstance(module, Block):
            raise HyenaB200Error("StepGraph: a residual input exists for a Block only")
        self.module, self.mixers = module, mixers
        self.caches = [cache.for_module(m) for m in mixers]
        # the position the graphs advance: the stack's (one for all its layers) or the operator's own
        self.cache = cache if isinstance(module, Backbone) or len(self.caches) > 1 else self.caches[0]
        B = cache.batch_size if batch_size is None else int(batch_size)
        if B != self.caches[0].batch_size:
            raise HyenaB200Error(f"StepGraph: batch size {B} differs from the decode cache's {self.caches[0].batch_size}")
        if any(m.filter_fn.bidirectional for m in mixers):
            raise HyenaB200Error("decoding needs a causal filter; this HyenaFilter is bidirectional")
        self.device = self.caches[0].h.device
        self.shape, self.dtype = (B, 1, mixers[0].d_model), dtype
        self.residual = residual
        self.res_dtype = (torch.float32 if module.residual_in_fp32 else dtype) if residual else None
        self._graphs, self._keys, self._side, self._scratch = {}, {}, None, []
        self._check_room()
        self._in = torch.zeros(self.shape, dtype=dtype, device=self.device)
        self._res = torch.zeros(self.shape, dtype=self.res_dtype, device=self.device) if residual else None
        self._graph(self.plan()[0])

    # ---------------------------------------------------------------------------------------- host planning
    def plan(self):
        """(route, refresh) of the next step: route "plain", "window" or "branch"; refresh when the window must be opened
        (decode_window_plan with the step count satisfied: a graph step never waits WINDOW_AFTER_STEPS steps)."""
        from . import ops
        c = self.caches[0]
        if c.branched:
            return "branch", False
        route = ops.decode_window_plan(c.t, c.lcap, ops.WINDOW_AFTER_STEPS, c.win_b, c.win_wc)
        return ("window", True) if route == "refresh" else (route, False)

    def _check_room(self):
        c = self.caches[0]
        if c.branched and c.t >= c.base + c.hc:
            raise HyenaB200Error(f"StepGraph: decoding past the branch horizon: position {c.t} is base + Hc = {c.base} + "
                                 f"{c.hc} (fork with a larger horizon, up to Lcap = {c.lcap})")
        if c.t >= c.lcap:
            raise HyenaB200Error(f"StepGraph: decoding past the cache: position {c.t} is Lcap = {c.lcap}")

    _READS = {"plain": ("k", "bias", "h", "tail", "s_t", "part", "pos"),
              "window": ("k", "bias", "h", "tail", "s_t", "part", "pos", "win_f"),
              "branch": ("k", "bias", "h", "tail", "s_t", "part", "pos", "f", "parent")}

    def _key(self, route):
        return tuple((id(x), x.data_ptr()) if x is not None else None
                     for c in self.caches for x in (getattr(c, n) for n in self._READS[route]))

    def _check_input(self, u_t, residual):
        for name, x, dt in (("input", u_t, self.dtype), ("residual", residual, self.res_dtype)):
            if x is None and dt is None:
                continue
            if x is None or dt is None:
                raise HyenaB200Error(f"StepGraph.step: this graph was captured {'with' if dt is not None else 'without'} "
                                     "a residual input")
            if tuple(x.shape) != self.shape or x.dtype != dt or x.device != self.device:
                raise HyenaB200Error(f"StepGraph.step: {name} {tuple(x.shape)} {x.dtype} on {x.device} differs from the "
                                     f"captured {self.shape} {dt} on {self.device}")

    # ---------------------------------------------------------------------------------------- stepping
    def step(self, u_t, residual=None):
        """One position: u_t (B, 1, D) -> the module's step output (a Block's is (hidden_states, residual)), in static
        tensors that the next step overwrites."""
        from . import ops
        self._check_input(u_t, residual)
        self._check_room()
        route, refresh = self.plan()
        if route in self._keys and self._key(route) != self._keys[route]:
            raise HyenaB200Error("StepGraph.step: a buffer of the decode cache was replaced since the capture (reallocated, "
                                 "re-forked or re-synced elsewhere); capture a new StepGraph")
        if refresh:
            for c in self.caches:
                ops.decode_window_refresh(c)
        graph, out = self._graph(route)
        c0 = self.caches[0]
        t = c0.t
        self.cache.sync_position()
        self._in.copy_(u_t)
        if residual is not None:
            self._res.copy_(residual)
        graph.replay()
        for c in self.caches:
            c.t += 1
            if not c.branched:
                c.steps += 1
        self.cache._pos_state.value = (t + 1, c0.win_b, c0.base)
        return out

    def _graph(self, route):
        """(graph, static output) of ``route``, captured on first use."""
        if route not in self._graphs:
            self._graphs[route] = self._capture(route)
            self._keys[route] = self._key(route)
        return self._graphs[route]

    def _run(self, route):
        """The step on the static inputs with the device-position kernels of ``route``, then the position advance."""
        from . import ops
        from .block import Backbone, Block
        if route == "plain":
            def core(p_t, ib, sw, sb, c):
                return ops.decode_step_dev(p_t, ib, sw, sb, c, min(c.lcap, ops.WINDOW_MIN_T))
        else:
            core = ops.decode_win_step_dev if route == "window" else ops.decode_branch_step_dev

        def mix(op, c):
            return lambda y: op._step_with(y, c, core)
        m = self.module
        with torch.no_grad():
            if isinstance(m, Backbone):
                hidden, res = self._in, None
                for layer, c in zip(m.layers, self.caches):
                    hidden, res = layer._run(hidden, res, mix(layer.mixer, c))
                y, _ = Block._add_norm(hidden, res, m.ln_f)
                out = y.to(hidden.dtype)
            elif isinstance(m, Block):
                out = m._run(self._in, self._res, mix(m.mixer, self.caches[0]))
            else:
                out = m._step_with(self._in, self.caches[0], core)
            ops.decode_pos_advance(self.cache.pos)
        return out

    def _capture(self, route):
        from . import ops
        caches, c0 = self.caches, self.caches[0]
        if route == "window":
            for c in caches:
                if c.win_f is None:           # the refresh writes it in place from now on (decode_window_refresh)
                    c.win_f = torch.zeros(c.order - 1, c.batch_size, c.d_model, ops.WINDOW, dtype=torch.float32,
                                          device=c.h.device)
        pos = self.cache.sync_position()
        # warm-up at the current position: the library's lazy set-up for the capturing stream (cuBLAS workspace, weight
        # images, module loading) happens here, not inside the capture.  A step writes g_t into h and shifts the tail:
        # both are restored.  The warm-up position keeps every route in bounds (window base t - t mod 4).
        j = c0.t - c0.base if c0.branched else c0.t
        saved = [(c.tail.clone(), c.h[..., j].clone()) for c in caches]
        warm = torch.tensor([c0.t, c0.t - c0.t % 4, c0.base], dtype=torch.int32)
        if self._side is None:
            self._side = torch.cuda.Stream(device=self.device)
        side = self._side
        side.wait_stream(torch.cuda.current_stream(self.device))
        # torch's streams are pooled, so the library's per-stream weight-image scratch of the capturing stream could be
        # replaced and freed by other work on it later: the graph gets scratch of its own, held here as long as it lives
        with ops.private_weight_images(self.device, side, self._scratch):
            with torch.cuda.stream(side):
                for _ in range(self.WARMUP):
                    pos.copy_(warm)
                    self._run(route)
                for c, (tail, col) in zip(caches, saved):
                    c.tail.copy_(tail)
                    c.h[..., j].copy_(col)
            torch.cuda.current_stream(self.device).wait_stream(side)
            self.cache._pos_state.value = None
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=side):
                out = self._run(route)
        return graph, out
