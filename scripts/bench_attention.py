"""Times the attention kernels alone (CUDA events, 30 launches after 3 warm-ups) and prints one JSON line:
  * forward at the 4B vision shape (B=64, S=197, H=24) with the relative-position bias as the dense (H,S,S_pad) table and in
    LUT form (the form the adapters use for S <= 384), outputs compared;
  * backward at the same shape with the dense bias / dbias tables and with the transposed tables the training stack uses
    (S <= 224), input gradients compared;
  * forward of 15 s audio (B=16, S=750) with the dense bias;
  * the call the inference stack makes (LUT form, ln_stats, no lse) at B=64 for S=33 (text), 197 (image) and 214 (text +
    image, two-segment LUT), with the rate against the bytes the algorithm has to move (qkv read, bf16 output and ln_stats
    records written).
usage: python scripts/bench_attention.py"""
import json
import sys

import torch

sys.path.insert(0, "."); sys.path.insert(0, "oracle")
from one_peace_b200 import kernels as K, relpos  # noqa: E402
import restated as R  # noqa: E402


def timeit(f, n=30):
    for _ in range(3):
        f()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        f()
    e1.record()
    torch.cuda.synchronize()
    return round(e0.elapsed_time(e1) / n * 1000, 1)


def maxrel(a, b):
    return float(((a.float() - b.float()).abs().max() / b.float().abs().max()).item())


res = {"gpu": torch.cuda.get_device_name()}
B, S, H = 64, 197, 24
D = H * 64
g = torch.Generator(device="cuda").manual_seed(0)
qkv = (torch.randn(B * S, 3 * D, device="cuda", generator=g) * 0.5).bfloat16()
bucket = R.make_image_bucket_position(14)
table = torch.randn(732, H, device="cuda", generator=g) * 0.5
li = relpos.build_lut_index(bucket.numpy(), relpos.image_codes(S, 14))
rp = K.RelPosBias(lut=K.relpos_lut_build(table, torch.from_numpy(li[0]).cuda()), code_row=torch.from_numpy(li[1]).cuda(),
                  code_col=torch.from_numpy(li[2]).cuda())
dense = K.relpos_bias_build(table, bucket.cuda(), S, H)
out = torch.empty(B * S, D, dtype=torch.bfloat16, device="cuda")
lse = torch.empty(B * H * S, device="cuda")
t_dense = timeit(lambda: K.attention(qkv, dense, None, B, S, H, out=out, lse=lse))
o_dense = out.clone()
t_lut = timeit(lambda: K.attention_tc(qkv, rp, None, B, S, H, out=out, lse=lse))
res["fwd_vision_us"] = {"dense_bias": t_dense, "lut_bias": t_lut, "max_rel_diff": maxrel(out, o_dense)}

d_out = torch.randn(B * S, D, device="cuda", generator=g).bfloat16()
dqkv = torch.zeros(B * S, 3 * D, dtype=torch.bfloat16, device="cuda")
dbias = torch.zeros_like(dense)
t_bd = timeit(lambda: K.attention_bwd(qkv, out, d_out, dense, None, lse, dqkv, dbias, B, S, H, 0.125))
dq_dense = dqkv.clone()
bias_t = K.relpos_bias_transpose(dense)
dbias_t = torch.zeros(H, K.BIAS_T_KEYS, K.BIAS_T_Q, device="cuda")
t_bt = timeit(lambda: K.attention_bwd_t(qkv, out, d_out, bias_t, None, lse, dqkv, dbias_t, B, S, H, 0.125))
res["bwd_vision_us"] = {"dense_tables": t_bd, "transposed_tables": t_bt, "dqkv_max_rel_diff": maxrel(dqkv, dq_dense)}

Ba, Sa = 16, 750
qa = (torch.randn(Ba * Sa, 3 * D, device="cuda", generator=g) * 0.5).bfloat16()
ba = R.make_token_bucket_position(256)[:Sa, :Sa]
da = K.relpos_bias_build(torch.randn(514, H, device="cuda", generator=g), ba.cuda(), Sa, H)
oa = torch.empty(Ba * Sa, D, dtype=torch.bfloat16, device="cuda")
res["fwd_audio_750_us"] = timeit(lambda: K.attention(qa, da, None, Ba, Sa, H, out=oa))


def stack_fwd(Sx, rpx):
    """LUT form with ln_stats and without lse, as the encoder stack calls it; us per launch and GB/s of algorithmic bytes"""
    qx = (torch.randn(B * Sx, 3 * D, device="cuda", generator=g) * 0.5).bfloat16()
    ox = torch.empty(B * Sx, D, dtype=torch.bfloat16, device="cuda")
    st = torch.empty(H * B * Sx * 2, device="cuda")
    us = timeit(lambda: K.attention_tc(qx, rpx, None, B, Sx, H, out=ox, ln_stats=st))
    nbytes = qx.numel() * 2 + ox.numel() * 2 + st.numel() * 4
    return {"us": us, "MB": round(nbytes / 1e6, 1), "GB_per_s": round(nbytes / us / 1e3, 1)}


def text_lut(Sx):
    li = relpos.build_lut_index(R.make_token_bucket_position(256)[:Sx, :Sx].numpy(), relpos.text_codes(Sx))
    return li, K.RelPosBias(lut=K.relpos_lut_build(torch.randn(514, H, device="cuda", generator=g), torch.from_numpy(li[0]).cuda()),
                            code_row=torch.from_numpy(li[1]).cuda(), code_col=torch.from_numpy(li[2]).cuda())


res["fwd_stack_us"] = {"S33_text": stack_fwd(33, text_lut(33)[1]), "S197_image": stack_fwd(S, rp)}
li17 = text_lut(17)[0]
rp214 = K.build_segmented_lut([(torch.randn(514, H, device="cuda", generator=g), li17, 17), (table, li, S)], "cuda")
res["fwd_stack_us"]["S214_two_segment"] = stack_fwd(17 + S, rp214)
print(json.dumps(res), flush=True)
