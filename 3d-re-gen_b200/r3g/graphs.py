"""CUDA-graph capture of the model forwards: the DiT step, the dense SDF decode, the VGGT aggregator, the camera head
and the DPT head each keep one GraphCache and replay its entries.

A graph replays into the addresses it was captured with, so an entry owns every buffer its kernels touch: the static
inputs, the outputs (allocated from the graph's private pool during capture) and the workspaces allocated before the
capture, passed as `keep`.  A model's workspace cache may then replace its buffers (another shape, an eager call) while
the graph stays cached: the entry still holds the captured ones."""
import torch

from . import _abi


class GraphEntry:
    def __init__(self, graph, inputs, outputs, launches, keep):
        self.graph = graph
        self.inputs = inputs        # static inputs: copy new values in before replay()
        self.outputs = outputs      # what the captured callable returned, rewritten by every replay()
        self.launches = launches    # r3g kernels in the graph (replays are not seen by r3g_launch_count)
        self.keep = keep

    def replay(self):
        self.graph.replay()


class GraphCache:
    """key -> GraphEntry.  With keep_all=False, capturing a new key drops the previous entry (and its buffers)."""

    def __init__(self, keep_all=False):
        self.keep_all = keep_all
        self.entries = {}

    def get(self, key, inputs, fn, keep=()):
        """The entry for `key`; if absent, `fn(*static inputs)` is run once as a warm-up (workspaces, lazily set
        function attributes) and then captured, both on a side stream of the inputs' device, whichever is current."""
        entry = self.entries.get(key)
        if entry is None:
            static = tuple(t.clone() for t in inputs)
            dev = static[0].device
            with torch.cuda.device(dev):
                side = torch.cuda.Stream(dev)
                side.wait_stream(torch.cuda.current_stream(dev))
                with torch.cuda.stream(side):
                    fn(*static)
                torch.cuda.current_stream(dev).wait_stream(side)
                ctx = _abi.get_context(dev.index)
                n0 = ctx.launches
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph, stream=side):
                    outputs = fn(*static)
                entry = GraphEntry(graph, static, outputs, ctx.launches - n0, keep)
            if not self.keep_all:
                self.entries.clear()
            self.entries[key] = entry
        return entry
