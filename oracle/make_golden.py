"""Generate tests/golden/*.npz from the REAL reference (container only).

    python -m oracle.make_golden

Imports the reference checkout named by $MEGATTS2_REFERENCE under oracle/stubs.py, loads the seeded weights of
oracle/weights.py into the reference's own modules (load_state_dict strict=True,
which also pins the state_dict key set), runs the reference functions on seeded
inputs, asserts that the restatement in oracle/ref_megatts2.py agrees, and writes
inputs + reference outputs as small fixtures.  The tests read only the fixtures.
"""
import json
import os
import sys
import warnings

import numpy as np
import torch
import torch.nn.functional as F

from . import ref_megatts2 as R
from . import stubs, weights

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def gen(seed):
    g = torch.Generator()
    g.manual_seed(seed)
    return g


def close(name, a, b, tol):
    a, b = a.detach().float(), b.detach().float()
    err = (a - b).abs().max().item() if a.numel() else 0.0
    scale = b.abs().max().item() if b.numel() else 0.0
    print(f"  {name:34s} max|d|={err:.3e}  (scale {scale:.3e})")
    assert err <= tol, f"{name}: oracle vs reference {err} > {tol}"


def save(name, **arrs):
    out = {}
    for k, v in arrs.items():
        if isinstance(v, torch.Tensor):
            v = v.detach().cpu().numpy()
        out[k] = v
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path} ({os.path.getsize(path) / 1024:.1f} KiB)")


def main():
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(8)
    warnings.simplefilter("ignore")
    G, plm, adm = stubs.build_reference_models()
    gsd, psd, asd = weights.g_state_dict(), weights.plm_state_dict(), weights.adm_state_dict()
    # strict load == the oracle's key/shape spec equals the reference's state_dict layout
    G.load_state_dict(gsd, strict=True)
    plm.load_state_dict(psd, strict=True)
    adm.load_state_dict(asd, strict=True)
    keys = {
        "G": {k: list(v.shape) for k, v in G.state_dict().items()},
        "plm": {k: list(v.shape) for k, v in plm.state_dict().items()},
        "adm": {k: list(v.shape) for k, v in adm.state_dict().items()},
    }
    with open(os.path.join(OUT, "state_dict_keys.json"), "w") as f:
        json.dump(keys, f, indent=0, sort_keys=False)
    gcfg, pcfg, acfg = weights.G_CFG, weights.PLM_CFG, weights.ADM_CFG
    g = R.SD(gsd)

    with torch.no_grad():
        # ---- a1 mel front end (through the reference's extract_mel_spec + stubbed wrapper)
        print("mel front end")
        from modules.tokenizer import extract_mel_spec  # type: ignore
        wav = torch.rand(3, 4000, generator=gen(1234)) * 2 - 1
        wav[2] *= 1e-7                                   # exercises the 1e-5 clamp floor
        ref = extract_mel_spec(wav)
        close("mel", R.mel_spectrogram(wav), ref, 2e-5)
        save("mel_frontend", wav=wav, mel=ref)

        # ---- a2 / C1: VQ prosody encoder, one 2-s clip + a ragged-length batch
        print("vqpe (C1)")
        mel1 = torch.randn(1, 125, 80, generator=gen(1235)) * 2 - 4
        zq, commit, vql, codes = G.vqpe(mel1)
        o_zq, o_commit, o_vql, o_codes, o_ze = R.vqpe_forward(g.sub("vqpe"), mel1, gcfg)
        assert torch.equal(codes, o_codes), "C1 codes differ"
        close("zq", o_zq, zq, 1e-5)
        close("vq_loss", o_vql, vql, 1e-5)
        assert commit.shape == o_commit.shape == (1, 1)
        ze_ref = G.vqpe.convnet(mel1[..., :20].transpose(1, 2))
        close("ze", o_ze, ze_ref, 1e-4)
        mel2 = torch.randn(2, 61, 80, generator=gen(1236)) * 2 - 4
        zq2, _, vql2, codes2 = G.vqpe(mel2)
        o2 = R.vqpe_forward(g.sub("vqpe"), mel2, gcfg)
        assert torch.equal(codes2, o2[3])
        close("zq ragged", o2[0], zq2, 1e-5)
        save("vqpe", mel1=mel1, codes1=codes, zq1=zq, ze1=ze_ref, vq_loss1=vql,
             mel2=mel2, codes2=codes2, zq2=zq2, vq_loss2=vql2)

        # ---- a4: VQ search incl. adversarial near-ties
        print("vq quantize")
        embed = gsd["vqpe.vq.vq.layers.0._codebook.embed"]
        cb = G.vqpe.vq.vq.layers[0]._codebook
        x = torch.randn(512, 256, generator=gen(1237))
        # points eps away from the midpoint of random code pairs, and exact codes
        ia = torch.randint(0, 1024, (256,), generator=gen(1238))
        ib = torch.randint(0, 1024, (256,), generator=gen(1239))
        mid = 0.5 * (embed[ia] + embed[ib])
        dirv = embed[ia] - embed[ib]
        eps = torch.logspace(-6, -2, 256).unsqueeze(1)
        x = torch.cat([x, mid + eps * dirv, mid - eps * dirv, embed[:64]], 0)
        idx = cb.quantize(x)
        assert torch.equal(idx, R.vq_quantize(x, embed))
        dec = G.vqpe.vq.decode(idx.view(1, 1, -1))
        close("vq decode", R.vq_decode(idx.view(1, 1, -1), embed), dec, 0)
        # fp64 distances, to tell genuine ties from rounding (used by the GPU test's slack)
        d64 = torch.cdist(x.double(), embed.double()).pow(2)
        top2 = d64.topk(2, largest=False).values
        save("vq_search", x=x, idx=idx, gap64=(top2[:, 1] - top2[:, 0]).float(), idx64=d64.argmin(-1))

        # ---- a6: encoder stacks (conv-FF and linear-FF), with and without masks
        print("transformer encoder")
        xe = torch.randn(2, 9, 512, generator=gen(1240))
        ref = G.mrte.phone_encoder(xe)
        o = R.encoder(g.sub("mrte.phone_encoder"), xe, 8, 2, True)
        close("phone_encoder", o, ref, 2e-4)
        xl = torch.randn(2, 7, 1024, generator=gen(1241))
        lens = torch.tensor([7, 7], dtype=torch.int32)
        ref_c = plm.plm(xl, lens, causal=True)
        close("plm encoder causal", R.encoder(R.SD(psd, "plm."), xl, 12, 16, False, lens=lens, causal=True), ref_c, 5e-4)
        ref_n = plm.plm(xl)
        close("plm encoder nomask", R.encoder(R.SD(psd, "plm."), xl, 12, 16, False), ref_n, 5e-4)
        save("encoder", x_phone=xe, y_phone=ref, x_plm=xl, y_plm_causal=ref_c, y_plm_nomask=ref_n)

        # ---- a5: MRTE.tc_latent
        print("mrte.tc_latent")
        phone = torch.randint(0, 320, (2, 12), generator=gen(1242))
        melp = torch.randn(2, 100, 80, generator=gen(1243)) * 2 - 4
        ref = G.mrte.tc_latent(phone, melp)
        o, o_ctx, o_px = R.mrte_tc_latent(g.sub("mrte"), phone, melp, gcfg)
        close("tc_latent", o, ref, 2e-4)
        ctx_ref = G.mrte.mel_encoder(melp.transpose(1, 2)).transpose(1, 2)
        close("mel_context", o_ctx, ctx_ref, 2e-4)
        save("mrte", phone=phone, mel=melp, tc_latent=ref, mel_context=ctx_ref)

        # ---- a8: LengthRegulator, incl. the reference's own test case (mrte.py:187-194)
        print("length regulator")
        lr_in = torch.randn(2, 10, 128, generator=gen(1244))
        d = torch.tensor([[1, 2, 3, 4], [1, 2, 3, 5]], dtype=torch.int32)
        from modules.mrte import LengthRegulator  # type: ignore
        lr = LengthRegulator(256, 16000, 16.0)
        ref = lr(lr_in[:, :4], d)
        assert ref.shape == (2, 11, 128)
        close("length_regulate", R.length_regulate(lr_in[:, :4], d), ref, 0)
        save("length_regulator", x=lr_in[:, :4], d=d, y=ref)

        # ---- a9: ADM.infer (batch 1 in the reference; two utterances)
        print("adm.infer")
        tcs = F.relu(torch.randn(2, 10, 512, generator=gen(1245)))
        raws, ints = [], []
        for b in range(2):
            # raw float trajectory: re-run the loop body through the reference modules
            p = torch.zeros(1, 1, 1)
            for t in range(10):
                x_emb = torch.cat([adm.tc_linear_emb(tcs[b:b + 1, :t + 1]), adm.dt_linear_emb(p)], -1)
                y = adm.predict_layer(adm.adm(adm.pos_emb(x_emb)))[:, -1:, :]
                p = torch.cat([p, y], 1)
            raws.append(p[:, 1:])
            ints.append(adm.infer(tcs[b:b + 1]))
        raw_ref, int_ref = torch.cat(raws), torch.cat(ints)
        o_int, o_raw = R.adm_infer(R.SD(asd), tcs, acfg, return_raw=True)
        close("adm raw", o_raw, raw_ref, 2e-3)
        assert torch.equal(o_int, int_ref), (o_int.flatten(), int_ref.flatten())
        print("   durations:", int_ref.flatten().tolist())
        dtok = torch.rand(2, 11, 1, generator=gen(1246)) * 20
        lens = torch.tensor([10, 10], dtype=torch.int32)
        fwd_ref, tgt_ref = adm(tcs, dtok, lens)
        o_fwd, o_tgt = R.adm_forward(R.SD(asd), tcs, dtok, lens, acfg)
        close("adm forward", o_fwd, fwd_ref, 2e-3)
        save("adm", tc_latent=tcs, raw=raw_ref, dur=int_ref, dtok=dtok, fwd=fwd_ref)

        # ---- a10: PLM.infer (free-running ids + per-step logits) and forward
        print("plm.infer")
        tc8 = F.relu(torch.randn(2, 12, 512, generator=gen(1247)))
        ids, lgs = [], []
        for b in range(2):
            ids.append(plm.infer(tc8[b:b + 1]))
            code = torch.tensor([[1024]])
            steps = []
            for t in range(12):     # teacher-forced on the reference's own ids
                x_emb = torch.cat([tc8[b:b + 1, :t + 1], plm.pc_embedding(code)], -1)
                lg = plm.predict_layer(plm.plm(plm.pos(x_emb)))[:, -1, :]
                steps.append(lg)
                code = torch.cat([code, ids[-1][:, t:t + 1]], 1)
            lgs.append(torch.stack(steps, 1))
        ids_ref, lg_ref = torch.cat(ids), torch.cat(lgs)
        o_ids, o_lg = R.plm_infer(R.SD(psd), tc8, pcfg, return_logits=True)
        assert torch.equal(o_ids, ids_ref), (o_ids, ids_ref)
        close("plm logits", o_lg, lg_ref, 2e-3)
        t2 = lg_ref.topk(2, -1).values
        print("   ids:", ids_ref[0].tolist(), " distinct:", ids_ref.unique().numel(),
              " min top-2 gap: %.3e" % (t2[..., 0] - t2[..., 1]).min().item())
        pcodes = torch.cat([torch.full((2, 1), 1024), ids_ref], 1)
        lens = torch.tensor([12, 12], dtype=torch.int32)
        f_ref, _ = plm(tc8, pcodes, lens)
        o_f, _ = R.plm_forward(R.SD(psd), tc8, pcodes, lens, pcfg)
        close("plm forward", o_f, f_ref, 2e-3)
        save("plm", tc8=tc8, ids=ids_ref, logits=lg_ref, fwd_logits=f_ref)

        # ---- 8f-1 (next row): opt-in causal decode, pinned on the reference's TRAINING forward (causal=True)
        print("causal decode (greedy / raw-feedback loops over the reference's teacher-forced forward)")
        codes = torch.full((2, 1), 1024, dtype=torch.int64)
        c_lgs = []
        for t in range(12):
            pc = torch.cat([codes, codes[:, :1]], 1)
            lg = plm(tc8[:, :t + 1], pc, torch.full((2,), t + 1, dtype=torch.int32))[0][:, -1]
            c_lgs.append(lg)
            codes = torch.cat([codes, lg.argmax(-1, keepdim=True)], 1)
        c_ids, c_lg = codes[:, 1:], torch.stack(c_lgs, 1)
        o_cids, o_clg = R.plm_infer_causal(R.SD(psd), tc8, pcfg, return_logits=True)
        assert torch.equal(o_cids, c_ids), (o_cids, c_ids)
        close("plm causal logits", o_clg, c_lg, 2e-3)
        # self-consistency: one teacher-forced pass over the decode's own output reproduces every step
        f_all, _ = plm(tc8, torch.cat([torch.full((2, 1), 1024), c_ids], 1), torch.tensor([12, 12], dtype=torch.int32))
        close("plm causal == teacher-forced", f_all, c_lg, 2e-3)
        t2 = c_lg.topk(2, -1).values
        print("   causal ids:", c_ids[0].tolist(), " differs from infer() at", int((c_ids != ids_ref).sum()), "of 24 positions;",
              " min top-2 gap: %.3e" % (t2[..., 0] - t2[..., 1]).min().item())
        p = torch.zeros(2, 1, 1)
        for t in range(10):
            dt_in = torch.cat([p, p[:, :1]], 1)
            y = adm(tcs[:, :t + 1], dt_in, torch.full((2,), t + 1, dtype=torch.int32))[0][:, -1]
            p = torch.cat([p, y.reshape(2, 1, 1)], 1)
        c_raw = p[:, 1:]
        c_dur = (c_raw + 0.5).to(torch.int32).clamp(1, 128)
        o_cdur, o_craw = R.adm_infer_causal(R.SD(asd), tcs, acfg, return_raw=True)
        close("adm causal raw", o_craw, c_raw, 2e-3)
        assert torch.equal(o_cdur, c_dur), (o_cdur.flatten(), c_dur.flatten())
        print("   causal durations:", c_dur.flatten().tolist())
        save("causal_decode", tc8=tc8, plm_ids=c_ids, plm_logits=c_lg, tc_latent=tcs, adm_raw=c_raw, adm_dur=c_dur)

        # ---- a12 + a14: the tensor-level body of Megatts.forward (models/megatts2.py:353-368)
        print("Megatts.forward body")
        phone = torch.randint(0, 320, (1, 6), generator=gen(1248))
        melp = torch.randn(1, 48, 80, generator=gen(1249)) * 2 - 4
        tc = G.mrte.tc_latent(phone, melp)
        dt = adm.infer(tc)[..., 0]
        dt_used = dt.clamp(max=6)            # keep the fixture small; the clamp is applied to both sides
        tc_exp = lr(tc, dt_used)
        tcp = F.max_pool1d(tc_exp.transpose(1, 2), 8, ceil_mode=True).transpose(1, 2)
        p_codes = plm.infer(tcp)
        zq = G.vqpe.vq.decode(p_codes.unsqueeze(0))
        zq = zq.transpose(1, 2).unsqueeze(2).contiguous().expand(-1, -1, 8, -1)
        zq = zq.reshape(1, -1, 256)
        xdec = torch.cat([tc_exp, zq[:, :tc_exp.shape[1], :]], -1).transpose(1, 2)
        mel_out = G.decoder(xdec)
        hsd = weights.hifigan_state_dict()
        o = R.synthesize(gsd, psd, asd, hsd, phone, melp, (gcfg, pcfg, acfg, weights.HIFIGAN_CFG),
                         forced_durations=dt_used)
        assert torch.equal(o["dt"], dt) and torch.equal(o["p_codes"], p_codes)
        close("e2e tc_latent", o["tc_latent"], tc, 2e-4)
        close("e2e mel", o["mel"], mel_out, 5e-4)
        print("   dt:", dt.flatten().tolist(), "p_codes:", p_codes.flatten().tolist())
        save("e2e", phone=phone, mel_prompt=melp, tc_latent=tc, dt=dt, dt_used=dt_used, p_codes=p_codes,
             mel=mel_out, wav_oracle=o["wav"])

        # ---- a13: HiFi-GAN restatement ("parity unpinned": oracle output only, for regression)
        print("hifigan (unpinned; oracle regression fixture)")
        melh = torch.randn(2, 80, 12, generator=gen(1250)) * 2 - 4
        wavh = R.hifigan_generator(hsd, melh, weights.HIFIGAN_CFG)
        assert wavh.shape == (2, 1, 256 * 22)
        save("hifigan", mel=melh, wav=wavh)
    print("all golden fixtures written")


if __name__ == "__main__":
    sys.exit(main())
