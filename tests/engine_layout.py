"""Test helpers: convert the engine's internal layouts (debug taps) to the reference's NCHW / OIHW, and the host rules
that choose the engine's launch plans, restated."""
import numpy as np
import torch

H100_SMS = 132


def geometry(args):
    h, w, cin = int(args.image_height), int(args.image_width), int(args.image_channels)
    geo = []
    for _ in range(int(args.num_stages)):
        geo.append(dict(h=h, w=w, cin=cin))
        h, w, cin = h // 2, w // 2, int(args.cnn_num_filters)
    return geo, (h, w)


# ----------------------------------------------------------------------------------------------------------------------
# the host rules of maml_b200_create / plan_chunks / tail_fusable, restated (engine.cu, kernels_tc.cu, kernels_bn.cu)
# ----------------------------------------------------------------------------------------------------------------------
def _tc_rpad(gw):
    return (128 + 2 * (gw + 1) + 7) // 8 * 8


def _tc_ring(F, gw):
    row = (F + 4) * 4
    extra = 128 * row + (128 // 2) * row              # split-K over 2 CTAs in tangent mode
    avail = 227 * 1024 - 4096 - 1024 - 4 * _tc_rpad(gw) * 128 - extra
    return min(8, avail // (2 * F * 128))


def host_plan(a, tasks, num_sms=H100_SMS):
    """The plan a handle made for ``tasks`` tasks (its max_tasks) takes, with the switches at their defaults:
      tc, ring: tensor-core convolutions / weight gradients for blocks l >= 1, and the depth of their ring next to split-K
                2 in tangent mode;
      tail:     the support pass's fused last block + head;
      chunks:   weight-gradient chunks per block l >= 1 (the most of any block);
      regime:   "latency" when one iteration's block-1 conv tiles (support + target, every task) fit one wave of SMs,
                else "throughput"; it decides programmatic dependent launch on the main chain (pdl) and the ring depth
                of the main-chain tensor-core convolutions (nb).
    The split-K cluster size of conv_tc_kernel comes from the occupancy calculator at launch and is not restated."""
    geo, _ = geometry(a)
    L, F = len(geo), int(a.cnn_num_filters)
    n_s = int(a.num_classes_per_set) * int(a.num_samples_per_class)
    n_t = int(a.num_classes_per_set) * int(a.num_target_samples)
    g1 = geo[1 if L > 1 else 0]
    G1 = (g1["h"] + 1) * (g1["w"] + 1)
    tiles = ((n_s * G1 + 127) // 128 + (n_t * G1 + 127) // 128) * tasks
    small = tiles <= num_sms
    rings = [_tc_ring(F, geo[l]["w"] + 1) for l in range(1, L)]
    tc = L > 1 and all(_tc_rpad(geo[l]["w"] + 1) <= 256 for l in range(1, L)) and min(rings) >= 2
    head_rows = 16 if n_s <= 16 else 4
    last = geo[-1]
    windows = n_s * ((last["h"] + 1) // 2) * ((last["w"] + 1) // 2)
    tail = n_s <= head_rows and windows <= 4 * (256 // (F // 4))
    chunks = []
    for l in range(1, L):
        rows = n_s * (geo[l]["h"] + 1) * (geo[l]["w"] + 1)
        nch = min(64, max(1, num_sms // (3 * tasks)), max(1, (rows + 15) // 16))
        rpc = ((rows + nch - 1) // nch + 15) // 16 * 16
        chunks.append((rows + rpc - 1) // rpc)
    return dict(tc=tc, tail=tail, ring=min(rings) if rings else None, chunks=max(chunks) if chunks else None,
                tiles=tiles, regime="latency" if small else "throughput", pdl=small, nb=8 if small else 4)


def norm_grid_regimes(a, tasks, num_sms=H100_SMS):
    """The regimes the grids of the normalisation kernels reach in one iteration (every block, support and target pass),
    from bn_grid / ln_grid (kernels_bn.cu) and the cap of the BatchNorm backward reduce (launch_bnbwd_reduce), which
    inner-loop BatchNorm always runs:
      ibn_reduce_capped: a BatchNorm pass needs more CTAs per task than num_sms, the reduce's cap;
      ibn_apply_capped:  it needs more than 4 * num_sms, bn_grid's cap (apply, forward and tangent kernels);
      ln_one_cta:        ln_grid's cap max(1, 4 * num_sms / (n * tasks)) is 1 and an image needs more;
      ln_capped:         that cap is above 1 and an image needs more."""
    geo, _ = geometry(a)
    F, N = int(a.cnn_num_filters), int(a.num_classes_per_set)
    wpb = 256 // (F // 4)
    out = set()
    for n in (N * int(a.num_samples_per_class), N * int(a.num_target_samples)):
        for gl in geo:
            per_img = ((gl["h"] + 1) // 2) * ((gl["w"] + 1) // 2)
            bx = (n * per_img + wpb - 1) // wpb
            if bx > num_sms:
                out.add("ibn_reduce_capped")
            if bx > 4 * num_sms:
                out.add("ibn_apply_capped")
            per_img_ctas = (per_img + wpb - 1) // wpb
            cap = max(1, 4 * num_sms // max(1, n * tasks))
            if per_img_ctas > cap:
                out.add("ln_one_cta" if cap == 1 else "ln_capped")
    return out


def device_sms():
    """The SM count the host rules see: the GPU's, or an H100's (132) on a machine without one."""
    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else H100_SMS


def traced_kernel_ids(m, batch, epoch):
    """The kernel ids (scripts/trace_kernel_ids.json) of one traced iteration, after an untraced one."""
    m.meta_gradient(batch, epoch)
    eng = m._engine
    eng.trace(True)
    m.meta_gradient(batch, epoch)
    tr = eng.trace_read(capacity=1 << 16)
    eng.trace(False)
    starts = [k for _, k, _ in tr if not (k & 0x80)]
    assert len(starts) == eng.last_launch_count()
    return set(starts)


# kernel ids of the device trace: the convolutions, the BatchNorm kernels of the plain path (bnact .. bnbwd_tan_fused,
# the fused tails, bnact_tan<GB>), and the layer-norm (primal, tangent) and inner-loop BatchNorm (PT: primal, tangent) ones
K_CONV_ROWS, K_WGRAD_ROW, K_CONV_TC, K_WGRAD_TC = 1, 3, 22, 27
K_BN = set(range(6, 14)) | {23, 24, 25, 32}
K_LN, K_LN_TAN = {33, 35, 37, 39, 41}, {34, 36, 38, 40, 42}
K_IBN, K_IBN_TAN = {43, 44, 45}, {46, 47, 48}


def check_norm_path(ids, norm, a, epoch, tasks):
    """The kernel ids of one iteration of a layer-norm (norm "ln") or inner-loop BatchNorm ("ibn") handle: that path's
    primal kernels, its tangent kernels exactly when the epoch is second order, none of the plain BatchNorm path's or the
    other path's, and the convolution kernels the host plan chooses."""
    own, own_tan, other = (K_LN, K_LN_TAN, K_IBN | K_IBN_TAN) if norm == "ln" else (K_IBN, K_IBN_TAN, K_LN | K_LN_TAN)
    second_order = bool(a.second_order) and epoch > a.first_order_to_second_order_epoch
    assert own <= ids, sorted(ids)
    assert (own_tan <= ids) if second_order else not (ids & own_tan), (second_order, sorted(ids))
    assert not ids & (K_BN | other), sorted(ids & (K_BN | other))
    plan = host_plan(a, tasks, device_sms())
    if plan["tc"]:
        assert {K_CONV_TC, K_WGRAD_TC} <= ids and not ids & {K_CONV_ROWS, K_WGRAD_ROW}, sorted(ids)
    elif int(a.num_stages) > 1:
        assert {K_CONV_ROWS, K_WGRAD_ROW} <= ids and not ids & {K_CONV_TC, K_WGRAD_TC}, sorted(ids)
    else:
        assert not ids & {K_CONV_ROWS, K_WGRAD_ROW, K_CONV_TC, K_WGRAD_TC}, sorted(ids)
    return plan


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
    """Internal fast-weight vector -> {reference name: tensor in reference layout}: per block W [3*3][Cin][F] and b (with
    inner-loop BatchNorm gamma / beta also beta, gamma [F]), then the linear layer [N][pix][F] and its bias."""
    geo, (ph, pw) = geometry(args)
    F, N = int(args.cnn_num_filters), int(args.num_classes_per_set)
    per_block = ("conv.bias", "norm_layer.bias", "norm_layer.weight") if args.enable_inner_loop_optimizable_bn_params \
        else ("conv.bias",)
    out, o = {}, 0
    v = np.asarray(vec)
    for l, g in enumerate(geo):
        cin = g["cin"]
        wsz = 9 * cin * F
        w = v[o:o + wsz].reshape(3, 3, cin, F).transpose(3, 2, 0, 1)     # [tap(ky,kx)][c][f] -> [f][c][ky][kx]
        out["classifier.layer_dict.conv%d.conv.weight" % l] = torch.from_numpy(np.ascontiguousarray(w))
        o += wsz
        for n in per_block:
            out["classifier.layer_dict.conv%d.%s" % (l, n)] = torch.from_numpy(v[o:o + F].copy())
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


def norm_params(args, state, theta, l, step):
    """Block l's normalisation scale / shift in one pass at inner step ``step``: BatchNorm gamma / beta [F] (the step's
    row with per-step statistics; the pass's fast weights ``theta`` with inner-loop gamma / beta), or layer norm's frozen
    weight and bias [F, h, w]."""
    from oracle import maml_oracle as O
    if getattr(args, "norm_layer", "batch_norm") == "layer_norm":
        _, _, gn, btn, _, _ = O.conv_names(l)
        return state[gn], state[btn]
    return O._bn_params(state, theta, args, l, step)


def activate_pool(zh, gamma, beta):
    """What the GPU computes from its normalised activations zh [n, F, h, w] (fp32), bit for bit:
    y = fmaf(gamma, zh, beta) (exact product + one rounding == fp64 evaluation rounded to fp32),
    a = y > 0 ? y : 0.01f * y (fp32), 2x2 max-pool first-max-wins in window order (what F.max_pool2d does on CPU).
    gamma / beta: [F] (BatchNorm) or [F, h, w] (layer norm).  Returns (leaky-ReLU slope per element, arg-max per pooling
    window, pooled output)."""
    import torch.nn.functional as Fnn
    shape = (1, -1, 1, 1) if gamma.dim() == 1 else (1,) + tuple(gamma.shape)
    y = (gamma.double().reshape(shape) * zh.double() + beta.double().reshape(shape)).float()
    slope = torch.where(y > 0, torch.ones_like(y), torch.full_like(y, 0.01))
    act = torch.where(y > 0, y, torch.tensor(0.01, dtype=torch.float32) * y)
    p, idx = Fnn.max_pool2d(act, 2, 2, return_indices=True)
    return slope, idx, p


def gpu_decisions(m, args, batch, epoch):
    """The discrete decisions the GPU actually took (leaky-ReLU branch per element, arg-max per pooling window) in every
    pass, reconstructed bit-exactly from the engine's normalised activations zh (``activate_pool``) and the pass's
    scale / shift (``norm_params``; inner-loop gamma / beta: the TASK's fast weights, theta^s in the support pass of step
    s, theta^{s+1} in its target pass).  ``m`` must have run ``meta_gradient`` with ``_debug_keep_target_passes`` set."""
    from oracle import maml_oracle as O
    a = args
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
        thetas = [theta_to_ref(eng.debug_read("theta", b, s, 0), a) for s in range(S + 1)] \
            if a.enable_inner_loop_optimizable_bn_params else [None] * (S + 1)
        for s in range(S):
            for kind, n, th in (("sup", N * K, thetas[s]), ("tgt", N * T, thetas[s + 1])):
                if kind == "tgt" and sched[s] is None:
                    continue
                per_layer = []
                for l, gl in enumerate(geo):
                    zh = grid_to_nchw(eng.debug_read(kind + "_zh", b, s, l), n, gl["h"], gl["w"], F)
                    slope, idx, _ = activate_pool(zh, *norm_params(a, sd, th, l, s))
                    per_layer.append((slope, idx))
                dec[(b, kind, s)] = per_layer
    return dec
