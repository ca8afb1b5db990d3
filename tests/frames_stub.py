"""A ``dropin.FrameStream`` without a device, for the host tests: only what ``submit``, ``submit_many`` and ``result``
read before they touch a device, with ``_launch`` recording each tick's slot, admitted frames and stream indices
instead of staging and running them."""
from improved_body_parts_b200 import dropin


def stream(input_stage="device", slots=2, track=None):
    fs = object.__new__(dropin.FrameStream)
    fs.input_stage, fs.device, fs._track = input_stage, 0, track
    fs.host_decodes, fs._next, fs._calls = 0, 0, 0
    fs._busy, fs._done, fs._held, fs.launched = [None] * slots, {}, {}, []

    def launch(slot, frames, streams):
        fs.launched.append((slot, frames, streams))
        return None, None

    fs._launch = launch
    fs._finish = lambda slot: None
    return fs


def keys(frames):
    """The tick key of a tick's admitted frames."""
    return tuple(f.key for f in frames)
