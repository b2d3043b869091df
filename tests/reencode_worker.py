"""Child process of tests/test_gpu_reencode.py (not a test file): runs the product's re-encoding on the device and
returns what it emitted.  The re-encoding kernels have no hardware record yet, so every case runs in a process of its
own under a timeout: a hang or a CUDA fault fails that one test and nothing else.

usage: python reencode_worker.py IN.pickle OUT.pickle     |     python reencode_worker.py errors
  IN:  dict(w, h, targets=[(y, u, v) ...], pred=[bytes ...], state=bytes, kf_q_weight, extra_frame_chunk)
  OUT: dict(frames=[bytes ...], in_step=bool)   in_step: a Decoder resumed from `state` that decodes the emitted frames
                                                equals Encoder::export_decoder() at the end
  IN a list of such dicts: OUT the list of their results, dict(error=str) where the library refused the case"""
import os
import pickle
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    a = pickle.load(open(sys.argv[1], "rb"))
    if isinstance(a, list):   # several cases: an error of the library is reported per case instead of ending the run
        from alfalfa_b200 import capi
        out = []
        for case in a:
            try:
                out.append(run(case))
            except (capi.Invalid, capi.Unsupported, capi.LogicError) as e:
                out.append({"error": "%s: %s" % (type(e).__name__, e)})
    else:
        out = run(a)
    pickle.dump(out, open(sys.argv[2], "wb"))


def run(a):
    from alfalfa_b200 import Context, Decoder, Encoder
    w, h = a["w"], a["h"]
    ctx = Context(w, h, max_frames=24)
    pred_decoder = Decoder(ctx)  # the prediction stream's own decoder (xc-enc.cc:254, 284-300)
    prediction_frames = []
    for c in a["pred"]:
        pf = pred_decoder.parse_frame(c, keep_labels=True)
        pred_decoder.decode_frame(pf)
        prediction_frames.append(pf)
    enc = Encoder.from_decoder(ctx, Decoder.deserialize(ctx, a["state"]))
    frames = enc.reencode(a["targets"], prediction_frames, a["kf_q_weight"], a["extra_frame_chunk"])
    rx = Decoder.deserialize(ctx, a["state"])
    for c in frames:
        rx.get_frame_output(c)
    in_step = rx == enc.export_decoder()
    del enc, rx, pred_decoder
    ctx.close()
    return {"frames": frames, "in_step": bool(in_step)}


def errors():
    import numpy as np
    import pytest
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from test_gpu_encoder import synth
    from alfalfa_b200 import Context, Decoder, Encoder, capi
    w, h = 64, 64
    ctx = Context(w, h, max_frames=12)
    enc = Encoder(ctx)
    y, u, v = synth(w, h, 0)
    key = enc.encode_with_quantizer(y, u, v, 40)
    inter = enc.encode_with_quantizer(*synth(w, h, 1), 40)
    d = Decoder(ctx)
    pk = d.parse_frame(key, keep_labels=True)
    d.decode_frame(pk)
    plain = Decoder(ctx)
    plain.decode_frame(plain.parse_frame(key))
    p_nolabels = plain.parse_frame(inter)
    pi = d.parse_frame(inter, keep_labels=True)
    with pytest.raises(capi.LogicError):
        enc.update_residues(y, u, v, pk)            # a key frame is not a prediction InterFrame
    with pytest.raises(capi.LogicError):
        enc.update_residues(y, u, v, p_nolabels)    # parsed without keep_labels
    with pytest.raises(capi.LogicError):
        Encoder(ctx).update_residues(y, u, v, pi)   # an Encoder without references
    with pytest.raises(capi.LogicError):
        enc.reencode_as_interframe(y, u, v, pi, 40)  # not a key frame
    with pytest.raises(capi.Unsupported):
        enc.write_frame(pi)                         # only key frames are written back unchanged
    assert enc.write_frame(pk) == key               # Frame::serialize of the parsed key frame = its own bytes
    assert len(enc.update_residues(y, u, v, pi)) > 0
    assert len(enc.reencode_as_interframe(y, u, v, pk, 44)) > 0
    ctx.close()
    print("ok")


if __name__ == "__main__":
    if sys.argv[1] == "errors":
        errors()
    else:
        main()
