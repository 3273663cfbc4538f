"""Dump what a step kernel computes on a seeded shape, so that the cluster step kernel (step2.cu) and the one-CTA-per-SM step
kernel (step.cu) -- or two builds of the library (PTTS_LIB) -- can be compared bit for bit: every step's logits and the tokens of a
free-running greedy run (one launch per step), and the tokens of an in-kernel top-k sampling run (many steps per launch).
Usage: python tools/cluster_bitwise.py dump OUT.npz {mini|h768} {cluster|legacy} [layers] [steps]
       python tools/cluster_bitwise.py compare A.npz B.npz"""
import os
import sys

import numpy as np

SHAPES = {"mini": {}, "h768": dict(hidden_size=768, num_attention_heads=12, ffn_dim=3072)}


def dump(out, shape, step, layers, steps):
    import torch
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import bench
    from parler_tts_b200 import DACConfig, ParlerTTSConfig, ParlerTTSDecoderConfig, ParlerTTSForConditionalGeneration
    os.environ["PTTS_STEP"] = step
    dev = torch.device("cuda", 0)
    B = 32
    mcfg = dict(bench.MINI, num_hidden_layers=layers, **SHAPES[shape])
    cfg = ParlerTTSConfig(vocab_size=32128, text_encoder={}, audio_encoder=DACConfig(), decoder=ParlerTTSDecoderConfig(**mcfg))
    model = ParlerTTSForConditionalGeneration(cfg, device=dev, dtype=torch.bfloat16)
    sd = bench.synthetic_state_dict(mcfg, dev, seed=7)
    for k in list(sd):   # livelier logits than the 0.02 init so that greedy decisions depend on the last bits
        if "lm_heads" in k:
            sd[k] = sd[k] * 10
    model.load_state_dict(sd)
    eng = model.decoder.engine
    enc, em, pr, pm = bench.synthetic_inputs(B, mcfg.get("hidden_size", 1024), 3, device=dev)
    L = steps + 2
    sess = eng.session(B, bench.P_LEN, bench.S_LEN, bench.P_LEN + L)
    sess.begin(L, do_sample=False)
    sess.prefill(pr, pm, enc, em)
    want = 2 if step == "cluster" else 1
    assert sess.fused == want, f"fused kind {sess.fused}, expected {want} ({step})"
    sess.sample()
    logits = []
    for _ in range(1, steps):
        sess.decode_forward()
        logits.append(sess.logits.float().cpu().numpy())
        sess.sample()
    greedy = sess.raw_ids[:, : steps + 1].cpu().numpy()
    sess.begin(L, do_sample=True, top_k=50, seed=1, min_new_tokens=steps, suppress_special=True, codebook_size=1024)
    sess.prefill(pr, pm, enc, em)
    sess.sample()
    sess.decode_steps(steps - 1)
    torch.cuda.synchronize()
    sampled = sess.raw_ids[:, : steps + 1].cpu().numpy()
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    np.savez(out, logits=np.stack(logits), greedy=greedy, sampled=sampled)
    print(f"{out}: {shape}, {step} step kernel, {len(logits)} logit steps, lib {os.environ.get('PTTS_LIB', '(product)')}, "
          f"logits finite: {bool(np.isfinite(np.stack(logits)).all())}")


def compare(a_path, b_path):
    a, b = np.load(a_path), np.load(b_path)
    ok = True
    for k in ("logits", "greedy", "sampled"):
        same = a[k].shape == b[k].shape and np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8))
        diff = float(np.abs(a[k].astype(np.float64) - b[k].astype(np.float64)).max()) if a[k].shape == b[k].shape else float("nan")
        print(f"{k}: {'bitwise identical' if same else 'DIFFERENT'} (shape {a[k].shape}, max |diff| {diff:g})")
        ok &= same
    print("BITWISE", "OK" if ok else "FAILED")
    return ok


if __name__ == "__main__":
    if sys.argv[1] == "dump":
        dump(sys.argv[2], sys.argv[3], sys.argv[4], int(sys.argv[5]) if len(sys.argv) > 5 else 4, int(sys.argv[6]) if len(sys.argv) > 6 else 40)
    else:
        sys.exit(0 if compare(sys.argv[2], sys.argv[3]) else 1)
