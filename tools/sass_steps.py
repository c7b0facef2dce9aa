#!/usr/bin/env python
"""Print one unrolled step of the hot loops from the built library's SASS, and the mnemonics that prove the asynchronous
staging (TMA bulk copy, cp.async, mbarrier) is in the shipped decoder.  Needs cuobjdump; no GPU.

    python tools/sass_steps.py [path/to/librans_b200.so]
"""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def functions(sass):
    out, name = {}, None
    for ln in sass.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            name = m.group(1)
            out[name] = []
        elif name:
            m = re.match(r"\s+/\*([0-9a-f]{4,5})\*/\s+(.*?);\s+/\*", ln)
            if m:
                out[name].append((m.group(1), m.group(2).strip()))
    return out


def step_between(instrs, opcode, skip, max_len=60):
    """Instructions from the `skip`-th occurrence of `opcode` to the next one (inclusive start, exclusive end)."""
    idx = [i for i, (_, s) in enumerate(instrs) if re.match(r"(@!?P\d+\s+)?" + re.escape(opcode), s)]
    pairs = [(a, b) for a, b in zip(idx, idx[1:]) if b - a < max_len]
    # the typical step: skip the first few (prologue copies), take the most common length, no control flow inside
    clean = [(a, b) for a, b in pairs[skip:] if not any(re.search(r"\b(BRA|BSSY|BSYNC|CALL|WARPSYNC|ENDCOLLECTIVE)\b", s) for _, s in instrs[a:b])]
    lengths = [b - a for a, b in clean]
    typical = max(set(lengths), key=lengths.count)
    a, b = next((a, b) for a, b in clean if b - a == typical)
    return instrs[a:b]


def main():
    lib = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "ryg_rans_b200", "librans_b200.so")
    fns = functions(subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout)
    dec = next(v for k, v in fns.items() if "block_decode_kernel" in k)
    enc = next(v for k, v in fns.items() if "word_encode_fused_kernelILb1ELb0ELb0E" in k)
    enc_gated = next(v for k, v in fns.items() if "word_encode_fused_kernelILb1ELb1ELb0E" in k)
    enc_varlen = next(v for k, v in fns.items() if "word_encode_fused_kernelILb1ELb1ELb1E" in k)
    tma = next(v for k, v in fns.items() if "word_decode_tma_kernel" in k and k.endswith("Lb0EEEvPKhmPKmPKjPhmjjPNS_10DecodeWorkEPjy"))
    ali = next(v for k, v in fns.items() if "alias_decode_persist_kernelILj16E" in k)
    tma_planned = next(v for k, v in fns.items() if "word_decode_planned_kernelILb0E" in k)
    ali_planned = next(v for k, v in fns.items() if "alias_decode_planned_kernelILj16E" in k)
    for title, step in (("word_decode_tma_kernel<DecShip, false> (round 2, shipped): one step (symbol store to symbol store)",
                         step_between(tma, "STG.E.U8", 2)),
                        ("word_decode_planned_kernel<false> (rb200_container_decode_async): one step (symbol store to symbol store)",
                         step_between(tma_planned, "STG.E.U8", 2)),
                        ("alias_decode_persist_kernel<16> (round 2, shipped): one step (symbol store to symbol store)",
                         step_between(ali, "STG.E.U8", 2)),
                        ("alias_decode_planned_kernel<16> (rb200_container_decode_async): one step (symbol store to symbol store)",
                         step_between(ali_planned, "STG.E.U8", 2)),
                        ("block_decode_kernel (round 1 window: decode_window_chunk with WordDecoder<false>): one step (vote to vote)",
                         step_between(dec, "VOTE.ANY", 5)),
                        ("word_encode_fused_kernel<R32>: one step (symbol load to symbol load)", step_between(enc, "LDS.U8", 8)),
                        ("word_encode_fused_kernel<R32, GATED> (rb200_container_model_encode_async): one step (symbol load to symbol "
                         "load)", step_between(enc_gated, "LDS.U8", 8)),
                        ("word_encode_fused_kernel<R32, GATED, GEOM> (rb200_container_model_encode_varlen_async): one step (symbol load "
                         "to symbol load)", step_between(enc_varlen, "LDS.U8", 8))):
        print("## %s: %d instructions" % (title, len(step)))
        print("```")
        for addr, ins in step:
            print("/*%s*/  %s" % (addr, ins))
        print("```")
        print()
    print("## Asynchronous staging in the shipped decoders (mnemonic: occurrences in the kernel)")
    print()
    for title, body in (("word_decode_tma_kernel<DecShip, false>", tma), ("alias_decode_persist_kernel<16>", ali)):
        counts = {}
        for _, ins in body:
            m = re.match(r"(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", ins)
            if m and re.match(r"(UBLKCP|LDGSTS|SYNCS|LDGDEPBAR|DEPBAR|ELECT|VOTE|ATOMG|REDG)", m.group(1)):
                counts[m.group(1)] = counts.get(m.group(1), 0) + 1
        print("* `%s` (%d instructions): %s" % (title, len(body), ", ".join("`%s` x %d" % kv for kv in sorted(counts.items()))))


if __name__ == "__main__":
    main()
