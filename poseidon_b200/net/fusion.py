"""Graph planning for the sm100 engine: which elementwise layers disappear into kernel epilogues.

* CONVOLUTION / INNER_PRODUCT followed by an in-place RELU  ->  ReLU fused into the GEMM epilogue, the
  RELU layer becomes a no-op;
* the ReLU *backward* mask of such a layer is applied by its consumers' backward kernels when every
  consumer can do so for free (LRN bwd, MAX-pool bwd, stride-1 conv dgrad epilogue) — otherwise the
  producer masks its incoming gradient itself (one extra elementwise pass);
* a data layer whose only consumer is a first-layer (C <= 4) convolution emits the padded NHWC4 layout
  that convolution's ROW-mode gather consumes, straight from the transform kernel.

The reference runs every layer as separate kernels (ReLU: layers/relu_layer.cu; bias: an extra GEMM in
conv_layer.cu:38-42); nothing there is fused.
"""
from __future__ import annotations

import logging

log = logging.getLogger("poseidon_b200")


def plan_sm100(net) -> None:
    from ..ops import sm100
    n = len(net.layers)
    net.skip_layer = [False] * n
    consumers = {}                       # blob name -> list of layer indices reading it
    for i, bn in enumerate(net.bottom_names):
        for b in bn:
            consumers.setdefault(b, []).append(i)

    # engine state (operand layouts) for every learnable layer
    fp8 = sm100.resolve_fp8(getattr(net.ctx, "fp8", None))
    scaling = sm100.resolve_fp8_scaling(getattr(net.ctx, "fp8_scaling", None), fp8)
    tail = "; scaling delayed" if scaling == "delayed" else ""
    for i, layer in enumerate(net.layers):
        if layer.type_name == "CONVOLUTION":
            cin = net.blob_shapes[net.bottom_names[i][0]][1]
            try:
                st = sm100.conv_state(layer, cin, fp8, scaling)
            except ValueError as e:
                raise ValueError(f"layer {net.layer_names[i]}: {e}") from e
            if fp8 == "fprop" and net.ctx.rank == 0:
                log.info("sm100 plan: conv %s: %s (%s)%s", net.layer_names[i], "fp8" if st.fp8 else "bf16", st.fp8_reason,
                         tail)
            elif fp8 == "fprop+dgrad" and net.ctx.rank == 0:
                log.info("sm100 plan: conv %s: %s (%s); dgrad %s (%s)%s", net.layer_names[i], "fp8" if st.fp8 else "bf16",
                         st.fp8_reason, "fp8" if st.fp8_dgrad else "bf16", st.fp8_dgrad_reason, tail)
            elif fp8 == "fprop+dgrad+wgrad" and net.ctx.rank == 0:
                log.info("sm100 plan: conv %s: %s (%s); dgrad %s (%s); wgrad %s (%s)%s", net.layer_names[i],
                         "fp8" if st.fp8 else "bf16", st.fp8_reason, "fp8" if st.fp8_dgrad else "bf16",
                         st.fp8_dgrad_reason, "fp8" if st.fp8_wgrad else "bf16", st.fp8_wgrad_reason, tail)
        elif layer.type_name == "INNER_PRODUCT" and getattr(layer, "_sm100", None) is None:
            layer._sm100 = sm100.IPState(layer, tuple(net.blob_shapes[net.bottom_names[i][0]]))

    # ReLU fusion
    for i, layer in enumerate(net.layers):
        if layer.type_name not in ("CONVOLUTION", "INNER_PRODUCT") or len(net.top_names[i]) != 1:
            continue
        top = net.top_names[i][0]
        nxt = [j for j in consumers.get(top, []) if j > i]
        if not nxt:
            continue
        j = nxt[0]
        relu = net.layers[j]
        if relu.type_name != "RELU" or net.top_names[j] != [top] or net.bottom_names[j] != [top]:
            continue
        # the in-place ReLU must be the first reader of the blob
        if any(k < j for k in nxt[1:]):
            continue
        slope = float(relu.slope)
        if layer.type_name == "INNER_PRODUCT":
            if slope != 0.0:
                continue
            layer.fused_relu = True
        else:
            layer.fused_relu_slope = slope
        net.skip_layer[j] = True
        # who applies the backward mask?
        if layer.type_name == "CONVOLUTION" and slope == 0.0 and layer.num_output % 8 == 0:
            # (consumers mask inside kernels that need channel counts in multiples of 8)
            readers = [k for k in nxt if k != j]
            ok = bool(readers)
            for k in readers:
                c = net.layers[k]
                if c.type_name == "LRN" and c.region == "ACROSS_CHANNELS":
                    continue
                if c.type_name == "POOLING" and c.method == "MAX" and len(net.top_names[k]) == 1:
                    continue
                if c.type_name == "CONVOLUTION" and c.stride == (1, 1) and not c._sm100.row_mode and \
                        len(net.bottom_names[k]) == 1:
                    continue
                ok = False
            if ok:
                layer._sm100.consumer_masks = True
                for k in readers:
                    c = net.layers[k]
                    if c.type_name == "CONVOLUTION":
                        c._sm100.mask_input = True
                    else:
                        c.engine_kw = dict(getattr(c, "engine_kw", {}), mask_input=True)

    # zero-copy CONCAT: bottoms produced by convolution kernels (ReLU fused or absent) and read by nobody else are
    # written straight into the concat output slab (channel-offset view with the slab's pixel pitch)
    producer_of = {}
    for i, tn in enumerate(net.top_names):
        for t in tn:
            producer_of[t] = i               # last writer (in-place layers overwrite)
    n_slab = 0
    for i, layer in enumerate(net.layers):
        if layer.type_name != "CONCAT" or layer.dim != 1 or len(net.bottom_names[i]) < 2:
            continue
        shapes = [net.blob_shapes[b] for b in net.bottom_names[i]]
        if any(s[1] % 8 for s in shapes) or len(set(net.bottom_names[i])) != len(net.bottom_names[i]):
            continue
        plan, off, ok = [], 0, True
        for b, shp in zip(net.bottom_names[i], shapes):
            writers = [j for j, tn in enumerate(net.top_names) if b in tn and not net.skip_layer[j]]
            readers = [j for j in consumers.get(b, []) if not net.skip_layer[j]]
            j = writers[-1] if writers else -1
            c = net.layers[j] if j >= 0 else None
            if c is None or len(writers) != 1 or c.type_name != "CONVOLUTION" or readers != [i] or \
                    getattr(c, "_concat_slab", None) is not None or c._sm100.Coutp != c._sm100.Cout:
                ok = False
                break
            plan.append((c, off, shp[1]))
            off += shp[1]
        if not ok:
            continue
        layer._slab_channels = off
        layer._slab_slices = {o: n_c for _, o, n_c in plan}
        for c, o, _ in plan:
            c._concat_slab = (layer, o)
        n_slab += 1
    if n_slab and net.ctx.rank == 0:
        log.info("sm100 plan: %d CONCAT layers are zero-copy (branch convolutions write into the concat slab)", n_slab)

    # data layer -> first conv hand-off
    for i, layer in enumerate(net.layers):
        if not getattr(layer, "is_data", False) or not net.top_names[i]:
            continue
        readers = consumers.get(net.top_names[i][0], [])
        if len(readers) == 1:
            c = net.layers[readers[0]]
            if c.type_name == "CONVOLUTION" and c._sm100.row_mode:
                layer.first_conv = c
    fused = sum(net.skip_layer)
    if fused and net.ctx.rank == 0:
        log.info("sm100 plan: %d ReLU layers fused into conv/IP epilogues", fused)
