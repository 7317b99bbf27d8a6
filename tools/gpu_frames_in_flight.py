"""Throughput of the bench workload with one frame at a time vs two frames in flight (megapose6d_b200/frame_pipeline.py),
over a sweep of reserved SMs.  Also checks that the pipelined results equal the sequential ones frame for frame.

    python tools/gpu_frames_in_flight.py --reserve 0,8,16,24,32 --steps 20 --out gpurun_out/frames_in_flight.json
"""
import argparse
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from megapose6d_b200 import frame_pipeline as FP  # noqa: E402
from megapose6d_b200.tensor_collection import PandasTensorCollection  # noqa: E402
from megapose6d_b200.types import ObservationTensor  # noqa: E402
from workloads import scenes  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reserve", default="0,8,16,24,32")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--slots", default="2")
    ap.add_argument("--priority", default="0,1")
    ap.add_argument("--conv-modes", default="8", help="comma-separated mpx_conv_set_mode values (set before building)")
    ap.add_argument("--out", type=Path, default=Path("gpurun_out/frames_in_flight.json"))
    args = ap.parse_args()
    sc = scenes.bench_scene(1)
    images, K, det_df = sc["images"].cuda(), sc["K"].cuda(), sc["det_df"]
    g = torch.Generator().manual_seed(7)
    pool = [(sc["bboxes"] + (0.0 if i == 0 else 1.0) * (4.0 * torch.rand(sc["bboxes"].shape, generator=g) - 2.0)).cuda()
            for i in range(4)]
    kw = dict(n_refiner_iterations=sc["n_refiner_iterations"], n_pose_hypotheses=sc["n_pose_hypotheses"])

    def frame(i):
        return ObservationTensor(images, K), PandasTensorCollection(det_df.copy(), bboxes=pool[i % len(pool)])

    def timed(fn):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

    rows = []
    import itertools
    import time
    variants = itertools.product([int(v) for v in args.reserve.split(",")], [int(v) for v in args.slots.split(",")],
                                 [{"0": None, "1": "high"}.get(v, v) for v in args.priority.split(",")], [int(v) for v in args.conv_modes.split(",")])
    from megapose6d_b200 import _abi
    for reserve, n_slots, prio, mode in variants:
        sms = FP.set_reserved_sms(reserve)
        _abi.lib().mpx_conv_set_mode(mode)
        ests = [scenes.build_estimator(sc) for _ in range(n_slots)]
        pipe = FP.FramePipeline(None, estimators=ests, tail_priority=prio)
        for est in ests:
            for i in range(5):
                est.run_inference_pipeline(*frame(i), **kw)
        torch.cuda.synchronize()
        # host cost of one frame: enqueue (submit) and bookkeeping (result) with an idle device
        t0 = time.perf_counter()
        pend = ests[0].submit_inference_pipeline(*frame(0), **kw)
        t1 = time.perf_counter()
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        pend.result()
        t3 = time.perf_counter()
        seq_out = []

        def run_seq():
            for i in range(args.steps):
                seq_out.append(ests[0].run_inference_pipeline(*frame(i), **kw)[0])

        pipe_out = []

        def run_pipe():
            for i in range(args.steps):
                done = pipe.submit(*frame(i), **kw)
                if done is not None:
                    pipe_out.append(done[0])
            pipe_out.extend(d[0] for d in pipe.drain())
            pipe.join()

        ms_seq = timed(run_seq)
        ms_pipe = timed(run_pipe)
        del seq_out[:], pipe_out[:]
        ms_seq2 = timed(run_seq)
        ms_pipe2 = timed(run_pipe)
        same = all(torch.equal(a.poses, b.poses) and a.infos["pose_logit"].tolist() == b.infos["pose_logit"].tolist()
                   for a, b in zip(seq_out, pipe_out)) and len(seq_out) == len(pipe_out) == args.steps
        rec = dict(conv_mode=mode, reserve_sms=reserve, sms_used=sms, slots=n_slots, tail_priority=prio, host_submit_ms=(t1 - t0) * 1e3,
                   host_result_ms=(t3 - t2) * 1e3, ms_per_frame_sequential=min(ms_seq, ms_seq2),
                   ms_per_frame_in_flight=min(ms_pipe, ms_pipe2), speedup=min(ms_seq, ms_seq2) / min(ms_pipe, ms_pipe2),
                   hyp_per_s_in_flight=576 / min(ms_pipe, ms_pipe2) * 1e3, results_identical=bool(same))
        print(json.dumps(rec), flush=True)
        rows.append(rec)
        del pipe, ests
        torch.cuda.empty_cache()
    FP.set_reserved_sms(0)
    args.out.parent.mkdir(parents=True, exist_ok=True)
    args.out.write_text(json.dumps(rows, indent=1))


if __name__ == "__main__":
    main()
