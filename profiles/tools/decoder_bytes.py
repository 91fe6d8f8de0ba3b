"""ONE byte / FLOP model of the SA-Open-1.0 Oobleck decoder for the fusion level the code implements
(friendly-stable-audio-tools_b200/csrc/oobleck.cu): used by bench.py (`oobleck_decoder` block of the JSON line) and by
profiles/tools/decoder_layer_table.py (per-layer table from an ncu launch list), so the two cannot disagree.

Every tensor-core convolution reads a 16-bit Snake-activated copy of its input (2 B) and writes the 16-bit activated
copy for its consumer (2 B); the un-activated skip stream of the ResidualUnits is `raw_bytes` wide (2 with fp16
operands since round 2, 4 = fp32 with bf16 or fp16x3 operands): written by the transposed convolution and by
the first two units of a stage, read by all three.  128- and 256-channel units are one fused launch (the conv7 ->
conv1 intermediate never leaves the SM); 512- and 1024-channel units are two launches.
"""

STRIDES = (8, 8, 4, 4, 2)
CHANNELS = (2048, 1024, 512, 256, 128, 128)
SURVEY_PER_RESUNIT_FUSED_FP32_GB = 16.41      # SURVEY.md 8(d): per-ResidualUnit-fused lower bound, fp32 activations
SURVEY_PER_CONV_FP32_GB = 34.83               # SURVEY.md 8(d): per-conv compulsory traffic, fp32 activations
DECODER_FLOPS_L1024 = 5.163e12                # SURVEY.md Appendix C


def layers(L, raw_bytes=2, fused=True):
    """[(name, flops, algorithmic bytes)] in launch order for L latent positions (one sample)."""
    r = raw_bytes
    out = [("ncl->nlc16", 0, 64 * L * (4 + 2)),
           ("conv_in k7 64->2048", 2 * L * 64 * 2048 * 7, L * (64 * 2 + 2048 * 2))]
    cin = CHANNELS[0]
    for s, cout in zip(STRIDES, CHANNELS[1:]):
        lo = L * s
        out.append((f"convT s{s} {cin}->{cout}", 2 * L * cin * cout * 2 * s, L * cin * 2 + lo * cout * (r + 2)))
        for j, d in enumerate((1, 3, 9)):
            wr = r if j < 2 else 0            # the last unit's raw value is not needed by anything
            if fused and cout in (128, 256):
                out.append((f"  resunit d{d} {cout} (fused)", 2 * lo * cout * cout * 8, lo * cout * (2 + r + wr + 2)))
            else:
                out.append((f"  conv7 d{d} {cout}", 2 * lo * cout * cout * 7, lo * cout * (2 + 2)))
                out.append((f"  conv1+skip {cout}", 2 * lo * cout * cout, lo * cout * (2 + r + wr + 2)))
        cin, L = cout, lo
    out.append(("conv_out k7 128->2", 2 * L * 128 * 2 * 7, L * (128 * 2 + 2 * 4)))
    return out


def totals(L=1024, raw_bytes=2, fused=True):
    ls = layers(L, raw_bytes, fused)
    return sum(f for _, f, _ in ls), sum(b for _, _, b in ls)


if __name__ == "__main__":
    for rb in (2, 4):
        f, b = totals(1024, rb)
        print(f"raw stream {rb} B: {f / 1e12:.3f} TFLOP, {b / 1e9:.2f} GB per sample of 1024 latents")
