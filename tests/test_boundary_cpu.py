"""CPU: the C-ABI library loads and exports every symbol the header declares; host-side logic that needs no GPU."""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    from xpretrain_b200 import _lib
    header = open(os.path.join(ROOT, "include", "xpretrain_b200.h")).read()
    declared = set(re.findall(r"\b(xp_[a-z0-9_]+)\s*\(", header))
    assert declared, "no declarations parsed"
    handle = _lib.lib()
    for name in declared:
        assert hasattr(handle, name), f"{name} declared in include/xpretrain_b200.h but not exported"
    assert declared == set(_lib.SIGNATURES), declared ^ set(_lib.SIGNATURES)
    assert handle.xp_version() == _lib.ABI_VERSION


_C_KINDS = {"int": "int32_t", "int32_t": "int32_t", "uint32_t": "uint32_t", "int64_t": "int64_t", "float": "float",
            "void": "void"}


def _c_kind(decl: str) -> str:
    """pointer / int32_t / uint32_t / int64_t / float / void of a C return type or parameter declaration."""
    if "*" in decl:
        return "pointer"
    words = [w for w in re.findall(r"\w+", decl) if w != "const"]
    return _C_KINDS.get(words[0], words[0])


def _py_kind(t) -> str:
    import ctypes as C
    if t is None:
        return "void"
    if t in (C.c_void_p, C.c_char_p) or issubclass(t, C._Pointer):
        return "pointer"
    return {C.c_int32: "int32_t", C.c_uint32: "uint32_t", C.c_int64: "int64_t", C.c_float: "float"}.get(t, t.__name__)


def _header_declarations():
    """({struct: [(field, kind)]}, {function: (return kind, [argument kinds])}, [enum names]) of the header, comments and
    preprocessor lines stripped.  An array field has the kind of its elements."""
    src = open(os.path.join(ROOT, "include", "xpretrain_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", " ", src, flags=re.S)
    src = "\n".join(line for line in src.splitlines() if not line.lstrip().startswith("#"))
    structs = {}
    for name, body in re.findall(r"typedef\s+struct\s+(\w+)\s*\{(.*?)\}\s*\1\s*;", src, flags=re.S):
        structs[name] = [(re.findall(r"\w+", part)[-1], "pointer" if "*" in part else _c_kind(decl))
                         for decl in body.split(";") if decl.strip()
                         for part in re.sub(r"\[[^\]]*\]", "", decl).split(",")]
    protos = {}
    for chunk in src.split(";"):
        m = re.search(r"\b(xp_\w+)\s*\(([^)]*)\)\s*$", chunk)
        if m:
            ret = re.split(r"[{}]", chunk[:m.start()])[-1]
            args = [a for a in m.group(2).split(",") if a.strip() not in ("", "void")]
            protos[m.group(1)] = (_c_kind(ret), [_c_kind(a) for a in args])
    enums = re.findall(r"\b(XP_(?:ACT|OUT|DTYPE)_\w+)\s*=", src)
    return structs, protos, enums


def test_declarations_match_the_header(tmp_path):
    """The hand-written ctypes declarations of _lib.py against include/xpretrain_b200.h, compiled by the host C compiler:
    every struct (the ctypes ones and the XpOptTensor numpy row) with the header's field names and kinds in order, its
    sizeof and each field's offset and size; the XP_ACT_* / XP_OUT_* / XP_DTYPE_* values and XP_ABI_VERSION; and for every
    prototype the return kind and each argument's kind (pointer / int32_t / uint32_t / int64_t / float).  A mismatch here hands a kernel
    wrong pointers or strides on the GPU.  Needs neither the built library nor a GPU; a missing C compiler is a failure
    (nvcc needs one to build this project)."""
    import ctypes as C
    import itertools
    import shutil
    import subprocess
    from xpretrain_b200 import _lib

    structs, protos, enums = _header_declarations()
    assert len(structs) >= 8 and len(protos) >= 50 and enums, "the header parse found too little"
    bad = []

    # the Python layouts: name -> (sizeof, {field: (offset, size)}, [(field, kind)] in order)
    layouts = {}
    for name, obj in vars(_lib).items():
        if isinstance(obj, type) and issubclass(obj, C.Structure) and obj is not C.Structure:
            layouts[name] = (C.sizeof(obj), {f: (getattr(obj, f).offset, getattr(obj, f).size) for f, _ in obj._fields_},
                             [(f, _py_kind(t._type_ if issubclass(t, C.Array) else t)) for f, t in obj._fields_])
    dt = _lib.XpOptTensor        # the numpy row keeps pointers as u8
    np_kinds = {"u8": "pointer", "i8": "int64_t", "i4": "int32_t", "f4": "float"}
    layouts["XpOptTensor"] = (dt.itemsize, {f: (dt.fields[f][1], dt.fields[f][0].itemsize) for f in dt.names},
                              [(f, np_kinds.get(dt.fields[f][0].base.str[1:], dt.fields[f][0].str)) for f in dt.names])
    if set(layouts) != set(structs):
        bad.append(f"structs declared on one side only: Python {sorted(set(layouts) - set(structs))}, "
                   f"header {sorted(set(structs) - set(layouts))}")
    py_consts = {n: getattr(_lib, n) for n in dir(_lib) if re.match(r"(ACT|OUT|DTYPE)_[A-Z0-9_]+$", n)}
    if {"XP_" + n for n in py_consts} != set(enums):
        bad.append(f"enum constants on one side only: {sorted({'XP_' + n for n in py_consts} ^ set(enums))}")
    py_consts["ABI_VERSION"] = _lib.ABI_VERSION

    # the C side: sizeof / offsetof / field sizes / enum values, printed by a program compiled against the header
    lines = []
    for s in sorted(set(layouts) & set(structs)):
        lines.append(f'printf("sizeof {s} %zu\\n", sizeof({s}));')
        for f in sorted(set(layouts[s][1]) & {f for f, _ in structs[s]}):
            lines.append(f'printf("field {s} {f} %zu %zu\\n", offsetof({s}, {f}), sizeof((({s}*)0)->{f}));')
    for n in sorted(py_consts):
        if n == "ABI_VERSION" or "XP_" + n in enums:
            lines.append(f'printf("value {n} %lld\\n", (long long)XP_{n});')
    prog = tmp_path / "abi_layout.c"
    prog.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "xpretrain_b200.h"\nint main(void) {\n  '
                    + "\n  ".join(lines) + "\n  return 0;\n}\n")
    cc = shutil.which(os.environ.get("CC", "cc"))
    assert cc, "no host C compiler (`cc`) found: nvcc needs one to build this project, and this test needs it too"
    exe = tmp_path / "abi_layout"
    r = subprocess.run([cc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, f"compiling the layout probe against the header failed:\n{r.stderr}"
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n")

    c_size, c_field, c_value = {}, {}, {}
    for line in filter(None, out):
        kind, *rest = line.split()
        if kind == "sizeof":
            c_size[rest[0]] = int(rest[1])
        elif kind == "field":
            c_field[rest[0], rest[1]] = (int(rest[2]), int(rest[3]))
        else:
            c_value[rest[0]] = int(rest[1])
    for s in sorted(set(layouts) & set(structs)):
        size, fields, order = layouts[s]
        for i, (py, h) in enumerate(itertools.zip_longest(order, structs[s])):
            if py != h:
                bad.append(f"{s} field {i}: (name, kind) {py} in Python, {h} in the header")
        if size != c_size[s]:
            bad.append(f"{s}: sizeof {size} in Python, {c_size[s]} in the header")
        for f in sorted(set(fields) & {f for f, _ in structs[s]}):
            if fields[f] != c_field[s, f]:
                bad.append(f"{s}.{f}: (offset, size) {fields[f]} in Python, {c_field[s, f]} in the header")
    for n, v in sorted(py_consts.items()):
        if n in c_value and c_value[n] != v:
            bad.append(f"XP_{n}: {v} in Python, {c_value[n]} in the header")

    # prototypes: the kind of the return value and of every argument
    if set(protos) != set(_lib.SIGNATURES):
        bad.append(f"functions declared on one side only: {sorted(set(protos) ^ set(_lib.SIGNATURES))}")
    for fn in sorted(set(protos) & set(_lib.SIGNATURES)):
        res, args = _lib.SIGNATURES[fn]
        py = (_py_kind(res), [_py_kind(a) for a in args])
        if py != protos[fn]:
            bad.append(f"{fn}: (return, arguments) {py} in Python, {protos[fn]} in the header")
    assert not bad, "the Python declarations disagree with include/xpretrain_b200.h:\n  " + "\n  ".join(bad)


def _stream_functions():
    """The header's functions whose last parameter is `void* stream`: the kernel launches."""
    src = open(os.path.join(ROOT, "include", "xpretrain_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", " ", src, flags=re.S)
    src = "\n".join(line for line in src.splitlines() if not line.lstrip().startswith("#"))
    out = set()
    for chunk in src.split(";"):
        m = re.search(r"\b(xp_\w+)\s*\(([^)]*)\)\s*$", chunk)
        if m and re.sub(r"\s+", " ", m.group(2).split(",")[-1]).strip() == "void* stream":
            out.add(m.group(1))
    return out


def test_every_launch_goes_through_ops_call():
    """ops._call is the one place a kernel is launched: it appends the current stream, and wrapping it sees every launch
    (test_gpu_stream_schedule.py delays chosen streams that way).  In the package's code (its syntax tree: docstrings,
    comments and error-message labels may name a function), every header function taking `void* stream` is reached only
    as the quoted first argument of `_call(...)` in ops.py, never as an attribute or through getattr; a launch function
    declared but never called is allowed.  No module other than ops.py and _lib.py calls or imports `lib`."""
    import ast
    launches = _stream_functions()
    assert len(launches) >= 40, f"the header parse found only {len(launches)} launch functions"
    pkg = os.path.join(ROOT, "xpretrain_b200")
    own = {os.path.join("xpretrain_b200", "ops.py"), os.path.join("xpretrain_b200", "_lib.py")}
    bad, used = [], set()
    for dirpath, _, files in os.walk(pkg):
        for f in sorted(files):
            if not f.endswith(".py"):
                continue
            path = os.path.join(dirpath, f)
            rel = os.path.relpath(path, ROOT)
            for node in ast.walk(ast.parse(open(path).read(), path)):
                where = f"{rel}:{getattr(node, 'lineno', 0)}"
                if isinstance(node, ast.Attribute) and node.attr in launches:
                    bad.append(f"{where}: .{node.attr} launched outside ops._call")
                if not isinstance(node, ast.Call):
                    if isinstance(node, ast.ImportFrom) and rel not in own and any(a.name == "lib" for a in node.names):
                        bad.append(f"{where}: imports lib")
                    continue
                fn = node.func.id if isinstance(node.func, ast.Name) else getattr(node.func, "attr", None)
                first = node.args[0] if node.args else None
                name = first.value if isinstance(first, ast.Constant) and isinstance(first.value, str) else None
                if fn == "_call" and rel == os.path.join("xpretrain_b200", "ops.py") and name in launches:
                    used.add(name)
                elif fn == "_call":
                    bad.append(f"{where}: _call outside ops.py or with no launch function name")
                if fn == "getattr" and len(node.args) > 1 and getattr(node.args[1], "value", None) in launches:
                    bad.append(f"{where}: getattr reaches {node.args[1].value}")
                if fn == "lib" and rel not in own:
                    bad.append(f"{where}: calls lib()")
    assert not bad, "launches that bypass ops._call:\n  " + "\n  ".join(bad)
    assert len(used) >= 40, f"only {len(used)} launch functions are called through ops._call"
    # the stream _call appends is the current one, as the last argument
    ops_src = open(os.path.join(pkg, "ops.py")).read()
    assert re.search(r"def _call\(name: str, \*args\) -> None:.*?getattr\(lib\(\), name\)\(\*args, "
                     r"torch\.cuda\.current_stream\(\)\.cuda_stream\)", ops_src, flags=re.S)
    assert len(re.findall(r"getattr\(lib\(\)", ops_src)) == 1
    print(f"\n{len(used)} of {len(launches)} launch functions called through ops._call; unused: {sorted(launches - used)}")


def test_no_cpu_fallback():
    """The product path must fail loudly off-GPU instead of computing on the host."""
    from clipvip_cases import b16, vidclip
    from xpretrain_b200 import _lib
    model = vidclip(b16(1, 1))
    with pytest.raises(_lib.XpError):
        model(video=torch.zeros(1, 1, 3, 224, 224), text_input_ids=torch.zeros(1, 4, dtype=torch.long),
              text_input_mask=torch.ones(1, 4, dtype=torch.long))


def test_product_path_never_imports_the_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "xpretrain_b200")):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dirpath, f)).read()
                assert "oracle" not in src.replace("# oracle", ""), os.path.join(dirpath, f)


def test_state_dict_names_match_reference_layout():
    from clipvip_cases import b16, vidclip
    from oracle import clipvip_oracle as O
    cfg = b16(2, 2)
    model = vidclip(cfg)
    sd = O.init_state_dict(cfg)      # keyed like the reference CLIPModel.state_dict() (pinned by make_golden.py)
    own = model.clipmodel.state_dict()
    assert set(own) == set(sd)
    for k in sd:
        assert own[k].shape == sd[k].shape and own[k].dtype == sd[k].dtype, k
    assert abs(float(model.clipmodel.logit_scale) - 4.6) < 1e-6
    # weight-decay grouping of the reference (optimization/utils.py:127) keys on these substrings
    names = [n for n, _ in model.named_parameters()]
    assert any(n.endswith("logit_scale") for n in names) and any("pre_layrnorm" in n for n in names)


def test_wgrad_plan_fills_waves():
    from xpretrain_b200.ops import wgrad_plan
    for n_out, n_in in [(3072, 768), (768, 3072), (2304, 768), (768, 768)]:
        bn, s = wgrad_plan(n_out, n_in, 150784)
        tiles = ((n_out + 127) // 128) * ((n_in + bn - 1) // bn) * s       # 128 x block_n tiles on the 132 SMs of an H100
        assert tiles / (-(-tiles // 132) * 132) > 0.9


def test_timesformer_module_has_the_reference_state_dict():
    """config #4 drop-in: parameter names/shapes of hd-vila/src/modeling/timesformer.py:421-455 (no kernel is called)."""
    from oracle import timesformer_oracle as TO
    from xpretrain_b200.modeling.timesformer import TimeSformer

    cfg = TO.TimeSformerCfg(depth=2, num_frames=7, H=10, W=16, embed_dim=128, num_heads=2)
    m = TimeSformer(depth=2, num_frames=7, H=10, W=16, embed_dim=128, num_heads=2)
    got = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert got == TO.param_shapes(cfg)
    m.load_state_dict(TO.init_state_dict(cfg, seed=0), strict=True)
    # reference init quirks (timesformer.py:457-464): temporal_fc of every block but the first starts at zero
    m2 = TimeSformer(depth=2, embed_dim=128, num_heads=2)
    assert float(m2.blocks[1].temporal_fc.weight.abs().sum()) == 0.0
    assert float(m2.blocks[0].temporal_fc.weight.abs().sum()) > 0.0
    import pytest
    import torch
    with pytest.raises(Exception):          # no CPU path
        m(torch.zeros(1, 7, 128, 10, 16))


def test_swin3d_module_has_the_reference_state_dict():
    """config #5 drop-in: parameters and buffers of LF-VILA/src/models/video_encoder.py:450-548 (no kernel is called)."""
    import torch
    from oracle import swin3d_oracle as SO
    from xpretrain_b200.modeling.swin3d import SwinTransformer3D

    cfg = SO.Swin3DCfg()
    m = SwinTransformer3D(patch_norm=True, local_window=8)              # the released VideoEncoder config is the default
    got = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert got == SO.param_shapes(cfg)
    sd = SO.init_state_dict(cfg, seed=0)
    m.load_state_dict(sd, strict=True)
    assert torch.equal(m.layers[2].blocks[0].attn.relative_position_index, SO.rel_pos_index(cfg.window_size[2]))
    assert sum(p.numel() for p in m.parameters()) == 89_229_448         # BASELINE.md §2


def test_init_weights_statistics_follow_the_reference():
    """CLIPPreTrainedModel._init_weights (CLIP_ViP.py:481-522, factor 1, initializer_range 0.02) + the ViP additions
    (`added_cls ~ N(0,1)` :153, `temporal_embedding = 0` :166): sample std of every tensor family within 3 % of the nominal."""
    import torch
    from xpretrain_b200.modeling.clip_vip import CLIPModel, ClipVipConfig
    torch.manual_seed(0)
    cfg = ClipVipConfig()
    m = CLIPModel(cfg)
    def std(t): return float(t.detach().float().std())
    def close(got, want): assert abs(got - want) < 0.03 * want, (got, want)
    ve, te = m.vision_model.embeddings, m.text_model.embeddings
    close(std(te.token_embedding.weight), 0.02); close(std(te.position_embedding.weight), 0.02)
    close(std(ve.patch_embedding.weight), 0.02); close(std(ve.position_embedding.weight), 0.02)
    assert abs(std(ve.class_embedding) - 768 ** -0.5) < 0.15 * 768 ** -0.5      # 768 samples only: wider band
    assert abs(std(ve.added_cls) - 1.0) < 0.1                           # N(0, 1), 3 x 768 samples
    assert float(ve.temporal_embedding.abs().max()) == 0.0
    for tower, tc in ((m.vision_model, cfg.vision), (m.text_model, cfg.text)):
        in_std = tc.hidden_size ** -0.5 * (2 * tc.num_hidden_layers) ** -0.5
        for layer in (tower.encoder.layers[0], tower.encoder.layers[-1]):
            for lin in (layer.self_attn.q_proj, layer.self_attn.k_proj, layer.self_attn.v_proj, layer.mlp.fc2):
                close(std(lin.weight), in_std)
            close(std(layer.self_attn.out_proj.weight), tc.hidden_size ** -0.5)
            close(std(layer.mlp.fc1.weight), (2 * tc.hidden_size) ** -0.5)
            for lin in (layer.self_attn.q_proj, layer.self_attn.out_proj, layer.mlp.fc1, layer.mlp.fc2):
                assert float(lin.bias.abs().max()) == 0.0
            for ln in (layer.layer_norm1, layer.layer_norm2):
                assert float((ln.weight - 1).abs().max()) == 0.0 and float(ln.bias.abs().max()) == 0.0
    close(std(m.visual_projection.weight), 768 ** -0.5); close(std(m.text_projection.weight), 512 ** -0.5)
    assert abs(float(m.logit_scale) - 4.60) < 1e-6


def test_training_restorer_shaped_checkpoint_round_trips(tmp_path):
    """E2E_TrainingRestorer (CLIP-ViP/src/utils/load_save.py:260-327): `restore.pt` = {'global_step', 'model_state_dict',
    'optim_state_dict'} with every fp32 tensor stored as CPU fp16 (`_to_cpu`, :177-192) and turned back into fp32 on load
    (`_to_cuda`, :159-174).  Our module tree and our AdamW must accept that file unchanged: same keys, same optimizer-state
    layout (`step`, `exp_avg`, `exp_avg_sq`; param_groups with lr / betas / eps / weight_decay / correct_bias)."""
    import torch
    from clipvip_cases import b16, vidclip
    from xpretrain_b200.optimization.adamw import AdamW, build_e2e_optimizer_w_lr_mul

    def to_cpu(state):     # restatement of load_save.py:177-192
        if isinstance(state, torch.Tensor):
            ret = state.cpu()
            return ret.half() if "Float" in state.type() else ret
        if isinstance(state, (list, tuple)):
            return type(state)(to_cpu(t) for t in state)
        if isinstance(state, dict):
            return {n: to_cpu(t) for n, t in state.items()}
        return state

    def to_f32(state):     # load_save.py:159-174 without the .cuda()
        if isinstance(state, torch.Tensor):
            return state.float() if "Half" in state.type() else state
        if isinstance(state, (list, tuple)):
            return type(state)(to_f32(t) for t in state)
        if isinstance(state, dict):
            return {n: to_f32(t) for n, t in state.items()}
        return state

    def build(seed):
        model = vidclip(b16(1, 1), seed=seed)
        opt = AdamW(build_e2e_optimizer_w_lr_mul(list(model.named_parameters()), 1e-4, 0.2), lr=1e-4, betas=(0.9, 0.98))
        return model, opt

    model, opt = build(0)
    g = torch.Generator().manual_seed(3)
    for group in opt.param_groups:                       # optimizer state in the reference layout (adamw.py:64-70)
        for p in group["params"]:
            opt.state[p] = {"step": 17, "exp_avg": torch.randn(p.shape, generator=g) * 1e-3,
                            "exp_avg_sq": torch.rand(p.shape, generator=g) * 1e-6}
    ckpt = {"global_step": 17, "model_state_dict": to_cpu(model.state_dict()), "optim_state_dict": to_cpu(opt.state_dict())}
    assert set(ckpt["optim_state_dict"]["param_groups"][0]) >= {"lr", "betas", "eps", "weight_decay", "correct_bias", "params"}
    path = tmp_path / "restore.pt"
    torch.save(ckpt, path)

    model2, opt2 = build(1)                              # different init: everything must come from the file
    loaded = torch.load(path, weights_only=False)
    model2.load_state_dict(to_f32(loaded["model_state_dict"]))
    opt2.load_state_dict(to_f32(loaded["optim_state_dict"]))
    for (n, a), (_, b) in zip(model.state_dict().items(), model2.state_dict().items()):
        want = a.half().float() if a.is_floating_point() else a
        assert torch.equal(b, want), n                   # fp16 storage is the reference's choice; the round trip adds nothing
        assert b.dtype == a.dtype
    for g1, g2 in zip(opt.param_groups, opt2.param_groups):
        assert {k: v for k, v in g1.items() if k != "params"} == {k: v for k, v in g2.items() if k != "params"}
        for p1, p2 in zip(g1["params"], g2["params"]):
            s1, s2 = opt.state[p1], opt2.state[p2]
            assert s2["step"] == 17 and s2["exp_avg"].dtype == torch.float32
            assert torch.equal(s2["exp_avg"], s1["exp_avg"].half().float())
            assert torch.equal(s2["exp_avg_sq"], s1["exp_avg_sq"].half().float())
    # load_state_dict_with_mismatch (load_save.py:86-115): shape-mismatched and unknown keys are skipped silently
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    sd["clipmodel.vision_model.embeddings.temporal_embedding"] = torch.zeros(1, 8, 768)
    sd["task_head.weight"] = torch.zeros(3)
    own = model2.state_dict()
    toload = {k: v for k, v in sd.items() if k in own and own[k].shape == v.shape}
    missing, unexpected = model2.load_state_dict(toload, strict=False)
    assert unexpected == [] and missing == ["clipmodel.vision_model.embeddings.temporal_embedding"]
