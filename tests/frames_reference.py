"""The reference the frame-stream GPU tests hold ``dropin.FrameStream`` to: ``dropin.predict`` followed by
``dropin.group`` on the same frame, with the wire record ``spg_group_batch`` writes for its maps.  None of it goes
through ``FrameStream``.

The network is a stand-in in the manner of test_gpu_predict_batch.py's: network-like maps keyed on the input size plus a
small term taken from the sample's own input, so that a frame read from the wrong slot changes its maps, and a sample's
output does not depend on its batch.  Its maps are built on its first call at a size, which is the frame stream's
warm-up, so the captured forward pass has no Python side effect and copies nothing from the host."""
import numpy as np

MODEL_PARAMS = dict(boxsize=160, stride=4, max_downsample=32, padValue=128)


class StandIn:
    def __init__(self, torch, synth, fixed=None):
        self.torch, self.synth, self._maps = torch, synth, dict(fixed or {})
        self.calls = 0

    def __call__(self, x):
        t = self.torch
        self.calls += 1
        n, Hp, Wp, _ = x.shape
        h, w = Hp // 4, Wp // 4
        if (h, w) not in self._maps:  # first call at a size: the warm-up, outside any capture
            self._maps[(h, w)] = t.from_numpy(self.synth.make_network_output(h * 1000 + w, h, w, 3, noise=0.0)).to(x.device)
        base = self._maps[(h, w)].repeat(n // 2, 1, 1, 1)
        own = x[:, ::4, ::4, :][..., t.arange(50, device=x.device) % 3].permute(0, 3, 1, 2)
        return [[base + own * 0.05]]


def _typed(v):
    if isinstance(v, (list, tuple)):
        return (type(v).__name__, [_typed(x) for x in v])
    return (type(v).__name__, repr(v))


def _reference(env, frame, params, model, input_stage="device", model_params=MODEL_PARAMS):
    """``dropin.predict`` + ``dropin.group``: the maps, process()'s people and the wire record spg_group_batch writes."""
    d, t = env.dropin, env.torch
    heat, paf = d.predict(frame, params, model, model_params, input_stage=input_stage)
    people = d.keypoints(*d.group(heat, paf, frame.shape[0], params)[3:])
    g = d._new_grouper(1)
    try:
        rec = t.zeros(g.wire_record_bytes(), dtype=t.uint8, device=env.dev)
        g.set_wire_output(rec.data_ptr())
        g.group_device(heat.tensor, paf.tensor, frame.shape[0], d._params(params), paf_as_f64=paf.as_f64)
        record = rec.cpu().numpy()
    finally:
        g.close()
    return heat, paf, people, record


def _live(env, record):
    """The bytes of a record the grouping writes: the header and the first n_persons rows."""
    n = int(env.wire.as_records(record, 17, env.dropin.CAP_ROWS)[0]["n_persons"])
    return bytes(record[:env.wire.HEADER_BYTES + n * (2 * 17 + 2) * 8])
