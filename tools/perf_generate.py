"""Decode-step cost of `FiD.generate` by number of beams, at the FiD-base decoder shape (12 decoder layers, d_model 768,
12 heads, 32 128 tokens) and n_context 40 x 384 keys per batch element (all keys live), bf16, synthetic weights.  The
encoder runs 2 layers: it runs once per generation and is not part of the per-step numbers.

For each batch size B and number of beams nb (nb = 1: greedy), min_length = max_length = 32 so every case decodes the same 31
steps, and the script reports:
  - ms per decode step under CUDA-graph replay and output tokens/s (B sequences advance one token per step).  One timed
    window holds --gens generations of 31 replays of the captured step each (with the state reset between generations, a
    few small fills); the median of --repeats windows is reported with the range;
  - the beam selection kernels' time per step (beam_topk + beam_select, the PROF_BEAM_SELECT hook, eager run);
  - the cross-attention kernel's time per step (the stream kernel at nb > 1, the decode kernel at nb = 1; eager run), the
    cross K|V bytes one step reads (live 64-key tiles x 64 keys x 2 (K, V) x H*64 x 2 B x layers: independent of nb) and
    both the kernel's and the whole step's achieved GB/s;
  - the card name and power limit, read in the same run.
--xkv 16,fp8 runs every case with the 16-bit and with the opt-in e4m3 cross K|V cache (FiD.generate(cross_kv_dtype="fp8"))
back to back (the fp8 bytes per step count the codes and the two fp32 scales per key and head), and prints the decode
state's cross K|V bytes at FiD-base and Atlas-xl dimensions (computed from the shapes).
One JSON line per case (and all of them to --out)."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

PROF_ATTENTION, PROF_DECODE_CROSS, PROF_BEAM_SELECT = 3, 5, 6


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return name, pl


def build_model(dev):
    import model_synth
    from atlas_b200.fid import FiD, T5ConfigLite

    over = dict(vocab_size=32128, num_layers=2, num_decoder_layers=12)
    cfg = {k: v for k, v in dict(model_synth.T5_CFG, **over).items()
           if k not in ("dropout_rate", "is_encoder_decoder", "use_cache")}
    model = FiD(T5ConfigLite(**cfg))
    sd, _ = model_synth.fill_state_dict(model.state_dict(), 202)
    model.load_state_dict(sd)
    return model.to(torch.bfloat16).to(dev).eval()


def profiled_ms(L, kind, fn, last):
    """Sum over the `last` event-bracketed launches of `kind` during fn() (eager) -> (ms, launches).  Taking the last ones
    leaves out the encoder's launches of the same kind, which run before the decode steps."""
    import ctypes

    L.atlas_b200_profile_enable(kind)
    fn()
    torch.cuda.synchronize()
    cap = 1 << 16
    ms = (ctypes.c_double * cap)()
    n = L.atlas_b200_profile_launches(ms, None, cap)
    L.atlas_b200_profile_collect(None, None)
    L.atlas_b200_profile_enable(0)
    picked = list(ms[:n])[-last:]
    return sum(picked), len(picked)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,8")
    ap.add_argument("--beams", default="1,2,4,8")
    ap.add_argument("--n-ctx", type=int, default=40)
    ap.add_argument("--text-len", type=int, default=384)
    ap.add_argument("--length", type=int, default=32)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--gens", type=int, default=10, help="generations per timed window")
    ap.add_argument("--xkv", default="16", help="cross K|V cache types to compare, e.g. 16,fp8")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "perf_generate measures the GPU: no device found"
    from atlas_b200._lib import lib
    from atlas_b200 import ops

    L = lib()
    dev = torch.device("cuda:0")
    name, power = card()
    model = build_model(dev)
    c = model.config
    H, nl, Lk = c.num_heads, c.num_decoder_layers, args.n_ctx * args.text_len
    steps = args.length - 1
    rows = []
    for B in [int(x) for x in args.batches.split(",")]:
        g = torch.Generator().manual_seed(5)
        ids = torch.randint(2, 32000, (B, Lk), generator=g).to(dev)
        mask = torch.ones(B, Lk, dtype=torch.bool, device=dev)
        model.encoder.config.n_context, model.encoder.config.bsz = args.n_ctx, B
        live_tiles = int(ops.key_block_live(((1.0 - mask.float()) * -1e9)).sum()) if ops._SKIP_MASKED else B * ((Lk + 63) // 64)
        for nb, xkv in [(int(x), k) for x in args.beams.split(",") for k in args.xkv.split(",")]:
            xkv = None if xkv == "16" else xkv
            # bytes of one key row per head: K and V, 64 values of 2 B each, or 64 e4m3 codes + a fp32 scale each
            xkv_bytes = live_tiles * 64 * 2 * H * (64 * 2 if xkv is None else 64 + 4) * nl
            kw = dict(max_length=args.length, min_length=args.length, num_beams=nb, cross_kv_dtype=xkv)

            def gen():
                with torch.no_grad():
                    return model.generate(input_ids=ids, attention_mask=mask, **kw)

            model.cuda_graphs = True
            out = gen()                                   # builds the state and captures the step graph
            torch.cuda.synchronize()
            states = model.__dict__["_decode_states"]
            key = (B, Lk, args.length, torch.bfloat16, dev) if nb == 1 else (B, Lk, args.length, torch.bfloat16, dev, nb)
            key = key + ((xkv,) if xkv is not None else ())
            st = states[key]
            def reset():
                if nb == 1:
                    st.seq.fill_(c.pad_token_id)
                    st.seq[:, 0] = c.decoder_start_token_id
                    st.tok_in.fill_(c.decoder_start_token_id)
                    st.done.zero_()
                    st.t_dev.zero_()
                else:
                    st.reset(c.decoder_start_token_id, c.pad_token_id)

            times = []
            for _ in range(args.repeats):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(args.gens):
                    reset()
                    for _ in range(steps):
                        st.graph.replay()
                b.record()
                torch.cuda.synchronize()
                times.append(a.elapsed_time(b) / (steps * args.gens))
            times.sort()
            ms_step = times[len(times) // 2]
            # eager runs with the profiler hook: the selection kernels and the cross-attention kernel per step
            model.cuda_graphs = False
            gen()
            sel_ms, sel_n = profiled_ms(L, PROF_BEAM_SELECT, gen, 2 * steps) if nb > 1 else (0.0, 0)
            x_ms, x_n = profiled_ms(L, PROF_ATTENTION if nb > 1 else PROF_DECODE_CROSS, gen, nl * steps)
            model.cuda_graphs = True
            row = dict(B=B, nb=nb, xkv=xkv or "16", n_ctx=args.n_ctx, text_len=args.text_len, steps=steps, ms_per_step=round(ms_step, 4),
                       ms_per_step_spread=[round(times[0], 4), round(times[-1], 4)],
                       tokens_per_s=round(B / (ms_step * 1e-3), 1), sequences_per_s=round(B / (ms_step * 1e-3 * steps), 2),
                       select_ms_per_step=round(sel_ms / steps, 4), select_launches=sel_n,
                       xattn_ms_per_step=round(x_ms / steps, 4), xattn_launches=x_n,
                       xkv_bytes_per_step=xkv_bytes, xattn_kernel_GBps=round(xkv_bytes / (x_ms / steps * 1e-3) / 1e9, 1),
                       step_GBps=round(xkv_bytes / (ms_step * 1e-3) / 1e9, 1), out_shape=list(out.shape),
                       card=name, power_limit=power)
            rows.append(row)
            print(json.dumps(row), flush=True)
    greedy = {(r["B"], r["xkv"]): r["ms_per_step"] for r in rows if r["nb"] == 1}
    for r in rows:
        if (r["B"], r["xkv"]) in greedy:
            r["step_vs_greedy"] = round(r["ms_per_step"] / greedy[(r["B"], r["xkv"])], 3)
    print(f"{name}, power limit {power}")
    print(f"{'B':>3} {'nb':>3} {'xKV':>4} {'ms/step':>8} {'x greedy':>8} {'tok/s':>9} {'select ms':>9} {'xattn ms':>8} "
          f"{'xKV MB':>8} {'xattn GB/s':>10} {'step GB/s':>9}")
    for r in rows:
        print(f"{r['B']:>3} {r['nb']:>3} {r['xkv']:>4} {r['ms_per_step']:>8.3f} {r.get('step_vs_greedy', 0):>8.2f} "
              f"{r['tokens_per_s']:>9.1f} "
              f"{r['select_ms_per_step']:>9.4f} {r['xattn_ms_per_step']:>8.3f} {r['xkv_bytes_per_step'] / 1e6:>8.1f} "
              f"{r['xattn_kernel_GBps']:>10.1f} {r['step_GBps']:>9.1f}")
    if "fp8" in args.xkv.split(","):
        # the decode state's cross K|V at B = 8, n_context 40 x 384 keys: FiD-base (12 layers, 12 heads) and Atlas-xl
        # dimensions (24 layers, d 2048 = 32 heads of 64)
        for label, layers, heads in (("FiD-base", 12, 12), ("Atlas-xl", 24, 32)):
            rows_kv = 8 * args.n_ctx * args.text_len
            b16 = rows_kv * 2 * heads * 64 * 2 * layers
            b8 = rows_kv * 2 * heads * (64 + 4) * layers
            print(f"decode-state cross K|V, {label} B=8: 16-bit {b16 / 1e9:.2f} GB, fp8 {b8 / 1e9:.2f} GB ({b8 / b16:.4f}x)")
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
