"""Test helpers: convert the engine's internal layouts (debug taps) to the reference's NCHW / OIHW."""
import numpy as np
import torch


def geometry(args):
    h, w, cin = int(args.image_height), int(args.image_width), int(args.image_channels)
    geo = []
    for _ in range(int(args.num_stages)):
        geo.append(dict(h=h, w=w, cin=cin))
        h, w, cin = h // 2, w // 2, int(args.cnn_num_filters)
    return geo, (h, w)


def grid_to_nchw(buf, n, h, w, F):
    """[n*(h+1)*(w+1), F] padded pixel grid (row 0 / column 0 of every image block are the shared zero padding)
    -> [n, F, h, w]."""
    a = np.asarray(buf).reshape(n, h + 1, w + 1, F)[:, 1:h + 1, 1:w + 1, :]
    return torch.from_numpy(np.ascontiguousarray(a.transpose(0, 3, 1, 2)))


def flat_to_nchw(buf, n, h, w, F):
    """[n, h*w, F] unpadded (last block's pooled output / features) -> [n, F, h, w]."""
    a = np.asarray(buf).reshape(n, h, w, F)
    return torch.from_numpy(np.ascontiguousarray(a.transpose(0, 3, 1, 2)))


def theta_to_ref(vec, args):
    """Internal fast-weight vector -> {reference name: tensor in reference layout}."""
    geo, (ph, pw) = geometry(args)
    F, N = int(args.cnn_num_filters), int(args.num_classes_per_set)
    out, o = {}, 0
    v = np.asarray(vec)
    for l, g in enumerate(geo):
        cin = g["cin"]
        wsz = 9 * cin * F
        w = v[o:o + wsz].reshape(3, 3, cin, F).transpose(3, 2, 0, 1)     # [tap(ky,kx)][c][f] -> [f][c][ky][kx]
        out["classifier.layer_dict.conv%d.conv.weight" % l] = torch.from_numpy(np.ascontiguousarray(w))
        o += wsz
        out["classifier.layer_dict.conv%d.conv.bias" % l] = torch.from_numpy(v[o:o + F].copy())
        o += F
    pix = ph * pw
    D = pix * F
    fw = v[o:o + N * D].reshape(N, pix, F).transpose(0, 2, 1).reshape(N, D)   # [k][pix][c] -> [k][c*pix + pix]
    out["classifier.layer_dict.linear.weights"] = torch.from_numpy(np.ascontiguousarray(fw))
    o += N * D
    out["classifier.layer_dict.linear.bias"] = torch.from_numpy(v[o:o + N].copy())
    return out


def rel_err(a, b):
    a, b = a.double(), b.double()
    return float((a - b).abs().max()) / max(float(b.abs().max()), 1e-30)


def gpu_decisions(m, g, batch, epoch):
    """The discrete decisions the GPU actually took (leaky-ReLU branch per element, arg-max per pooling
    window), reconstructed bit-exactly from the engine's normalised activations zh:
    y = fmaf(gamma, zh, beta) (exact product + one rounding == fp64 evaluation rounded to fp32),
    a = y > 0 ? y : 0.01f * y (fp32), first-max-wins in window order (what F.max_pool2d does on CPU).
    ``m`` must have run ``meta_gradient`` with ``_debug_keep_target_passes`` set."""
    import torch.nn.functional as Fnn
    from oracle import maml_oracle as O
    a = g.args
    eng = m._engine
    geo, _ = geometry(a)
    F = int(a.cnn_num_filters)
    N, K, T = int(a.num_classes_per_set), int(a.num_samples_per_class), int(a.num_target_samples)
    S = int(a.number_of_training_steps_per_iter)
    B = batch[0].shape[0]
    sched = O.target_pass_schedule(a, epoch, True, S)
    sd = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    dec = {}
    for b in range(B):
        for s in range(S):
            for kind, n in (("sup", N * K), ("tgt", N * T)):
                if kind == "tgt" and sched[s] is None:
                    continue
                per_layer = []
                for l, gl in enumerate(geo):
                    zh = grid_to_nchw(eng.debug_read(kind + "_zh", b, s, l), n, gl["h"], gl["w"], F)
                    _, _, gn, btn, _, _ = O.conv_names(l)
                    gam, bet = (sd[gn][s], sd[btn][s]) if a.per_step_bn_statistics else (sd[gn], sd[btn])
                    y = (gam.double()[None, :, None, None] * zh.double() + bet.double()[None, :, None, None]).float()
                    slope = torch.where(y > 0, torch.ones_like(y), torch.full_like(y, 0.01))
                    act = torch.where(y > 0, y, torch.tensor(0.01, dtype=torch.float32) * y)
                    _, idx = Fnn.max_pool2d(act, 2, 2, return_indices=True)
                    per_layer.append((slope, idx))
                dec[(b, kind, s)] = per_layer
    return dec
