"""Replays of the shared-memory images the per-sample kernels consume (no GPU): the image of a blob is walked exactly like the
kernel walks it, and the GEMVs it encodes are compared with the dense matrices of the model.  Used by the CPU tests of the
default model (test_host_logic.py) and of the stress models (test_stress_models.py)."""
import ctypes
import numpy as np


def int8_image(L, blob):
    """(return code, image bytes, layout words) of lpcnet_b200_debug_image (int8 kernel)."""
    out = np.zeros(256 * 1024, np.uint8)
    lay = np.zeros(24, np.uint32)
    L.lpcnet_b200_debug_image.argtypes = [ctypes.c_char_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    r = L.lpcnet_b200_debug_image(blob, len(blob), out.ctypes.data, out.size, lay.ctypes.data)
    return r, out, lay


def float_image(L, blob):
    """(return code, image bytes, layout words) of lpcnet_b200_debug_image_n (neuron-per-lane float kernel)."""
    out = np.zeros(300000, np.uint8)
    lay = np.zeros(32, np.uint32)
    L.lpcnet_b200_debug_image_n.argtypes = [ctypes.c_char_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    r = L.lpcnet_b200_debug_image_n(blob, len(blob), out.ctypes.data, out.size, lay.ctypes.data)
    return r, out, lay


def dense_from_sparse(w, idx, nrows, ncols, block):
    """Dense [nrows][ncols] matrix of a block-sparse array (printSparseVector, dump_lpcnet.py:83-117); block(w32) -> [8 rows][4 cols]."""
    M = np.zeros((nrows, ncols), w.dtype)
    p = wp = 0
    for rg in range(nrows // 8):
        nb = idx[p]; p += 1
        for _ in range(nb):
            pos = idx[p]; p += 1
            M[rg * 8:rg * 8 + 8, pos:pos + 4] = block(w[wp:wp + 32]); wp += 32
    return M


def list_lengths(idx):
    """Block count of every 8-row group of an index array."""
    p, out = 0, []
    while p < len(idx):
        out.append(int(idx[p])); p += int(idx[p]) + 1
    return out


def xs_offset(c, s):
    return c * 128 + (((((s >> 4) & 1) << 6) | ((s & 7) << 3)) ^ (((c & 1) << 6) | ((c & 2) << 4))) + ((s >> 3) & 1) * 4


def replay_int8_image(L, blob, arrs, na=384):
    """Walks the int8 image like sample_kernel.cu (warp -> slot -> gate -> list of quads = MMA operands; (row group, K part) for
    the GRU_B input GEMV) and checks, for random u8 inputs, that the integer GEMVs equal the dense int8 matrices of `arrs`; that every
    neuron group is owned once; the order of each warp's lists (r0 h0 r1 h1 ... | z0 z1 ...); the (su-)biases, diagonals, GRU_B
    recurrent weights and dual_fc rows; and the readable slack behind every array.  Returns what the walk saw."""
    r, img, lay = int8_image(L, blob)
    assert r > 0, "image refused"
    wA, metaA, wB, metaB, image_bytes, total, nA, nB, SM_IMAGE, PARA, DIRA, GRPA, DIRB, WBREC, PARB, FCW, NWC, GPW, FCN, KP, NA, FAST = [int(v) for v in lay[:22]]
    assert r == image_bytes and NA == na and NWC * GPW * 8 == na
    assert total == SM_IMAGE + image_bytes and total <= 227 * 1024 and FCN in (8, 16, 32, 64)
    img = img[:image_bytes]
    rel = lambda o: o - SM_IMAGE
    ngrp = na // 8
    i8block = lambda w: w.reshape(8, 4)                                       # int8 blob block = [8 out][4 in]
    MA = dense_from_sparse(arrs["sparse_gru_a_recurrent_weights"].astype(np.int64), arrs["sparse_gru_a_recurrent_weights_idx"], 3 * na, na, i8block)
    MB = dense_from_sparse(arrs["gru_b_weights"].astype(np.int64), arrs["gru_b_weights_idx"], 48, na, i8block)
    x = np.random.default_rng(0).integers(0, 256, na).astype(np.int64)

    def replay_quads(wq, mq, q0, nq):
        """sum over quads q0..q0+nq of W[8 out][slot][4 in] . x[column block of the slot]; also counts the slots whose class
        (c & 3) repeats inside a quad and the padding slots (all-zero weights)"""
        acc = np.zeros(8, np.int64); clash = pad = 0
        for q in range(q0, q0 + nq):
            classes = set()
            for t in range(4):
                e = int(mq[q, t]); c = e >> 7
                assert e == xs_offset(c, 0) and c < na // 4
                classes.add(c & 3)
                pad += int(not wq[q, :, t, :].any())
                acc += wq[q, :, t, :] @ x[4 * c:4 * c + 4]
            clash += 4 - len(classes)
        return acc, clash, pad

    dirA = img[DIRA:DIRA + NWC * GPW * 3 * 2 * 4].view(np.uint32).reshape(NWC, GPW, 3, 2)
    grpA = img[GRPA:GRPA + NWC * GPW * 4].view(np.uint32).reshape(NWC, GPW)
    parA = img[PARA:PARA + NWC * GPW * 3 * 16 * 4].view(np.float32).reshape(NWC, GPW, 3, 2, 8)
    wAi = img[rel(wA):rel(wA) + nA * 128].view(np.int8).astype(np.int64).reshape(nA, 8, 4, 4)     # [quad][out][slot][in]
    mA = img[rel(metaA):rel(metaA) + nA * 8].view(np.uint16).reshape(nA, 4)
    assert sorted(grpA.reshape(-1).tolist()) == list(range(ngrp))            # every neuron group owned exactly once
    assert int(dirA[:, :, :, 1].sum()) == nA
    subias, diag = arrs["sparse_gru_a_subias"].reshape(2, 3 * na)[1], arrs["sparse_gru_a_recurrent_weights_diag"]
    got = np.zeros(3 * na, np.int64)
    loads, rh_stream, clashes, padA = [], [], 0, 0
    for w in range(NWC):
        # the warp's lists are contiguous and in the order the kernel walks them (first quad of the warp = r of slot 0)
        q = int(dirA[w, 0, 1, 0])
        for sl in range(GPW):
            for gate in (1, 2):
                assert int(dirA[w, sl, gate, 0]) == q
                q += int(dirA[w, sl, gate, 1])
        rh_stream.append(q - int(dirA[w, 0, 1, 0]))
        for sl in range(GPW):
            assert int(dirA[w, sl, 0, 0]) == q
            q += int(dirA[w, sl, 0, 1])
        loads.append(q - int(dirA[w, 0, 1, 0]))
        for sl in range(GPW):
            g = int(grpA[w, sl])
            for gate in range(3):
                q0, nq = int(dirA[w, sl, gate, 0]), int(dirA[w, sl, gate, 1])
                acc, cl, pd = replay_quads(wAi, mA, q0, nq)
                got[gate * na + 8 * g:gate * na + 8 * g + 8] += acc; clashes += cl; padA += pd
                np.testing.assert_array_equal(parA[w, sl, gate, 0], subias[gate * na + 8 * g:gate * na + 8 * g + 8])
                np.testing.assert_array_equal(parA[w, sl, gate, 1], diag[gate * na + 8 * g:gate * na + 8 * g + 8])
    np.testing.assert_array_equal(got, MA @ x)

    dirB = img[DIRB:DIRB + 6 * KP * 2 * 4].view(np.uint32).reshape(6, KP, 2)
    assert int(dirB[:, :, 1].sum()) == nB
    wBi = img[rel(wB):rel(wB) + nB * 128].view(np.int8).astype(np.int64).reshape(nB, 8, 4, 4)
    mB = img[rel(metaB):rel(metaB) + nB * 8].view(np.uint16).reshape(nB, 4)
    gotB = np.zeros(48, np.int64)
    clashesB = padB = 0
    for rg in range(6):
        for part in range(KP):
            acc, cl, pd = replay_quads(wBi, mB, int(dirB[rg, part, 0]), int(dirB[rg, part, 1]))
            gotB[rg * 8:rg * 8 + 8] += acc; clashesB += cl; padB += pd
    np.testing.assert_array_equal(gotB, MB @ x)
    # GRU_B recurrent block layout [out/8][in/4][8][4] and su-biases; dual_fc rows of the upper tree levels
    np.testing.assert_array_equal(img[WBREC:WBREC + 768].view(np.int8), arrs["gru_b_recurrent_weights"])
    np.testing.assert_array_equal(img[PARB:PARB + 96 * 4].view(np.float32), arrs["gru_b_subias"].reshape(-1))
    fcw = img[FCW:FCW + FCN * 36 * 4].view(np.float32).reshape(FCN, 36)
    np.testing.assert_array_equal(fcw[:, :32], arrs["dual_fc_weights"].reshape(256, 32)[:FCN])
    np.testing.assert_array_equal(fcw[:, 32:34], arrs["dual_fc_bias"].reshape(2, 256).T[:FCN])
    np.testing.assert_array_equal(fcw[:, 34:36], arrs["dual_fc_factor"].reshape(2, 256).T[:FCN])
    # readable slack: the pipelined GEMVs read up to 4 quads of weights and 6 meta entries past the end of a stream
    assert metaA - wA >= (nA + 4) * 128 and wB - metaA >= (nA + 6) * 8 and metaB - wB >= (nB + 4) * 128 and total - metaB >= (nB + 6) * 8
    return dict(nA=nA, nB=nB, loads=loads, rh_stream=rh_stream, clashes=clashes, clashesB=clashesB, padA=padA, padB=padB,
                fcw_nodes=FCN, fast_cvt=FAST, total=total, nwc=NWC, kparts=KP, partsB=dirB[:, :, 1].copy(), grpA=grpA.copy())


def replay_float_image(L, blob, arrs, na=384):
    """Walks the image of the neuron-per-lane float kernel (sample_kernel_f32n.cu) and checks: every compute lane owns one neuron,
    the fp16 blocks transposed to [8 rows][4 cols] reproduce the dense float matrices (the weights are fp16-exact), the biases,
    diagonals and dual_fc rows, the `dense` flag (set only when every GRU_B list is the full row in order) and the slack behind
    every array.  Returns the GRU_B chain each of the two GRU_B warps takes (dense / uniform / general) and the dense flag."""
    r, out, lay = float_image(L, blob)
    assert r > 0, "image refused"
    wA, metaA, wB, metaB, image_bytes, total, nA, nB, IMG, NEUR, DIRA, PARA, DIRB, PARB, WBREC, FCW, dense, NA = [int(v) for v in lay[:18]]
    assert r == image_bytes and total <= 227 * 1024 and total == IMG + image_bytes and NA == na
    img = out[:image_bytes]
    rel = lambda o: o - IMG
    fblock = lambda w: w.reshape(4, 8).T                                      # float blob block = [4 cols][8 rows]
    MA = dense_from_sparse(arrs["sparse_gru_a_recurrent_weights"].astype(np.float64), arrs["sparse_gru_a_recurrent_weights_idx"], 3 * na, na, fblock)
    MB = dense_from_sparse(arrs["gru_b_weights"].astype(np.float64), arrs["gru_b_weights_idx"], 48, na, fblock)
    neur = img[NEUR:NEUR + 2 * na].view(np.uint16)
    assert sorted(neur.tolist()) == list(range(na))                           # every neuron owned by exactly one lane
    assert all((neur[8 * k:8 * k + 8] == neur[8 * k] + np.arange(8)).all() and neur[8 * k] % 8 == 0 for k in range(na // 8))
    dirA = img[DIRA:DIRA + na // 8 * 3 * 2 * 4].view(np.uint32).reshape(na // 8, 3, 2)
    blkA = img[rel(wA):rel(wA) + nA * 64].view(np.float16).astype(np.float64).reshape(nA, 8, 4)
    mA = img[rel(metaA):rel(metaA) + nA * 2].view(np.uint16)
    got = np.zeros((3 * na, na))
    nxt = 0
    for g in range(na // 8):
        for q in range(3):
            b0, nb = int(dirA[g, q, 0]), int(dirA[g, q, 1])
            assert b0 == nxt; nxt += nb                                       # lists in blob order (group, gate), contiguous
            for b in range(b0, b0 + nb):
                pos = int(mA[b]) // 4
                assert mA[b] % 16 == 0
                got[q * na + 8 * g:q * na + 8 * g + 8, pos:pos + 4] += blkA[b]
    np.testing.assert_array_equal(got, MA)
    dirB = img[DIRB:DIRB + 48].view(np.uint32).reshape(6, 2)
    blkB = img[rel(wB):rel(wB) + nB * 64].view(np.float16).astype(np.float64).reshape(nB, 8, 4)
    mB = img[rel(metaB):rel(metaB) + nB * 2].view(np.uint16)
    gotB = np.zeros((48, na))
    in_order = True
    for rg in range(6):
        b0, nb = int(dirB[rg, 0]), int(dirB[rg, 1])
        in_order &= nb == na // 4
        for k, b in enumerate(range(b0, b0 + nb)):
            pos = int(mB[b]) // 4
            in_order &= pos == 4 * k
            gotB[rg * 8:rg * 8 + 8, pos:pos + 4] += blkB[b]
    np.testing.assert_array_equal(gotB, MB)
    assert dense == int(in_order)                                            # dense flag: offsets are 16 * block index
    para = img[PARA:PARA + 6 * na * 4].view(np.float32).reshape(3, 2, na)
    np.testing.assert_array_equal(para[:, 0], arrs["sparse_gru_a_bias"][1].reshape(3, na))
    np.testing.assert_array_equal(para[:, 1], arrs["sparse_gru_a_recurrent_weights_diag"].reshape(3, na))
    fcw = img[FCW:FCW + 256 * 36 * 4].view(np.float32).reshape(256, 36)
    np.testing.assert_array_equal(fcw[:, :32], arrs["dual_fc_weights"].reshape(256, 32))
    # slack: the pipelined chains read up to 4 blocks / 8 meta entries past a list
    assert metaA - wA >= (nA + 4) * 64 and wB - metaA >= (nA + 8) * 2 and metaB - wB >= (nB + 4) * 64 and total - metaB >= (nB + 8) * 2
    # GRU_B chain of compute warps 0 and 1 (sample_kernel_f32n.cu): lane cl walks row cl % 48; one chain per warp, chosen from the
    # list lengths of its 32 rows and the dense flag
    lens = dirB[:, 1].astype(int)
    chains = []
    for w in (0, 1):
        n = [lens[((w * 32 + l) % 48) >> 3] for l in range(32)]
        chains.append(("dense" if dense else "uniform") if min(n) == max(n) else "general")
    return dict(dense=dense, chains=chains, nB=nB)
