"""The library's launch rules, read from csrc/ (no GPU):
- every kernel launch goes through Launch (common.cuh): no raw <<<>>> and no cudaLaunchKernelEx anywhere else;
- a kernel reached by a PDL launch (Launch::pdl) begins with pdl_enter(), whose griddepcontrol.wait holds it until its predecessor is
  done -- without it the kernel races its predecessor;
- a kernel whose body calls pdl_enter() is launched with PDL, or the wait is wasted.
A PDL launch names its kernel directly (k_name or k_name<...>), or as the `kernel` argument of the callback it sits in, passed to a
for_each_* selector; then every kernel that selector names counts as reached.  Any other kernel expression (a table, a local variable) is
reported: its kernels cannot be read."""
import re
import shutil
from pathlib import Path

CSRC = Path(__file__).resolve().parent.parent / "gaussiansplats3d_b200" / "csrc"
LAUNCHER = "common.cuh"


def _sources(csrc):
    return {p.name: re.sub(r"//[^\n]*", "", p.read_text()) for p in sorted(csrc.glob("*.cu*")) + sorted(csrc.glob("*.h"))}


def _close(text, i, open_ch="(", close_ch=")"):
    """Index of the bracket closing the one at text[i]."""
    depth = 0
    for k in range(i, len(text)):
        depth += text[k] == open_ch
        depth -= text[k] == close_ch
        if depth == 0:
            return k
    raise ValueError("unbalanced brackets")


def _top_level_args(text):
    args, depth, cur = [], 0, ""
    for ch in text:
        depth += ch in "([{"
        depth -= ch in ")]}"
        if ch == "," and depth == 0:
            args.append(cur.strip())
            cur = ""
        else:
            cur += ch
    return args + [cur.strip()]


def kernel_bodies(csrc=CSRC):
    """{kernel name: body text} of every __global__ function."""
    out = {}
    for text in _sources(csrc).values():
        for m in re.finditer(r"__global__\s+void\s+(?:__launch_bounds__\s*\([^)]*\)\s*)?(\w+)\s*\(", text):
            brace = text.index("{", _close(text, m.end() - 1))
            out[m.group(1)] = text[brace + 1:_close(text, brace, "{", "}")]
    return out


def selectors(csrc=CSRC):
    """{for_each_* name: kernels its body names}"""
    out = {}
    for text in _sources(csrc).values():
        for m in re.finditer(r"static\s+void\s+(for_each_\w+)\s*\(", text):
            brace = text.index("{", _close(text, m.end() - 1))
            out[m.group(1)] = set(re.findall(r"\b(k_\w+)\s*<", text[brace:_close(text, brace, "{", "}")]))
    return out


def pdl_launches(csrc=CSRC):
    """[(file, kernel expression, kernels it reaches)] of every Launch::pdl call."""
    sel = selectors(csrc)
    out = []
    for name, text in _sources(csrc).items():
        for m in re.finditer(r"\.pdl\s*\(", text):
            kernel = _top_level_args(text[m.end():_close(text, m.end() - 1)])[1]
            direct = re.fullmatch(r"(k_\w+)\s*(<.*>)?", kernel)
            if direct:
                reached = {direct.group(1)}
            else:   # the callback argument of the innermost for_each_* call whose argument list holds the launch; anything else is unresolved
                spans = [(c.group(1), c.end() - 1, _close(text, c.end() - 1))
                         for c in re.finditer(r"\b(for_each_\w+)\s*(?:<[^;{}]*>)?\s*\((?=\s*\[)", text[:m.start()])]
                inside = [sp for sp in spans if sp[1] < m.start() < sp[2]]
                reached = sel.get(inside[-1][0], set()) if inside and kernel == "kernel" else set()
            out.append((name, kernel, reached))
    return out


def violations(csrc=CSRC):
    found = []
    for name, text in _sources(csrc).items():
        if name == LAUNCHER:
            continue
        for what in ("<<<", "cudaLaunchKernelEx"):
            if what in text:
                found.append(f"{name}: a raw {what} launch outside the launcher")
    bodies = kernel_bodies(csrc)
    reached = set()
    for name, kernel, ks in pdl_launches(csrc):
        if not ks:
            found.append(f"{name}: PDL launch of {kernel!r}: no kernel found for it")
        reached |= ks
    for k in sorted(reached):
        if k not in bodies:
            found.append(f"{k}: launched with PDL but not defined")
        elif not re.sub(r"static_assert\s*\([^;]*\);", "", bodies[k]).lstrip().startswith("pdl_enter();"):   # (compile-time checks run nothing)
            found.append(f"{k}: launched with PDL but does not begin with pdl_enter()")
    for k, body in sorted(bodies.items()):
        if "pdl_enter()" in body and k not in reached:
            found.append(f"{k}: calls pdl_enter() but is never launched with PDL")
    return found


def test_every_launch_follows_the_launch_rules():
    assert violations() == []


def test_the_rules_see_the_frame_chain():
    """The reading finds the kernels it is meant to: the selectors' kernels and the radix scatters among the PDL launches."""
    reached = set().union(*(ks for _, _, ks in pdl_launches()))
    assert {"k_depth", "k_project", "k_blend", "k_radix_scatter", "k_bucket", "k_raster_init"} <= reached
    assert not {"k_peer_signal", "k_peer_release", "k_peer_wait_release", "k_peer_wait_arrived"} & reached
    assert len([k for k, b in kernel_bodies().items() if "pdl_enter()" in b]) == 18


def _mutated(tmp_path, file, old, new):
    """A copy of csrc/ with `old` replaced by `new` once in `file`."""
    dst = tmp_path / "csrc"
    shutil.copytree(CSRC, dst, ignore=shutil.ignore_patterns("*.so", "*.o"))
    text = (dst / file).read_text()
    assert text.count(old) == 1, old
    (dst / file).write_text(text.replace(old, new))
    return dst


def test_a_pdl_launch_of_a_kernel_without_the_wait_is_caught(tmp_path):
    csrc = _mutated(tmp_path, "raster_kernels.cuh", "launch.plain(nullptr, k_peer_signal,", "launch.pdl(nullptr, k_peer_signal,")
    assert violations(csrc) == ["k_peer_signal: launched with PDL but does not begin with pdl_enter()"]


def test_a_pdl_launch_through_a_table_is_caught(tmp_path):
    """gs_compute_distances picks its kernel from a table: made a PDL launch, it is reported, not credited to a selector elsewhere."""
    csrc = _mutated(tmp_path, "engine.cu", "Launch(st).plain(nullptr, kernels[integer][dyn],", "Launch(st).pdl(nullptr, kernels[integer][dyn],")
    assert violations(csrc) == ["engine.cu: PDL launch of 'kernels[integer][dyn]': no kernel found for it"]


def test_a_raw_launch_is_caught(tmp_path):
    csrc = _mutated(tmp_path, "engine.cu", "Launch(e->stream).plain(nullptr, k_flush_l2, e->sm_count * 8, 512, 0, e->flush.p, words, ++tick);",
                    "k_flush_l2<<<e->sm_count * 8, 512, 0, e->stream>>>(e->flush.p, words, ++tick);")
    assert violations(csrc) == ["engine.cu: a raw <<< launch outside the launcher"]
