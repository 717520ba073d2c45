"""Command layer: `semtools search` / `semtools workspace` (reference src/cmds/search.rs,
src/cmds/workspace.rs, src/json_mode.rs, flags of src/bin/semtools.rs:52-83,12-27) on top of
the H100 library.  Output is reproduced byte for byte: header
`{file}:{start}::{end} ({distance})`, `{:4}: {line}` 1-based numbering, TTY highlight,
serde_json pretty printing, Rust float Display (shortest round-trip, never scientific)."""
from __future__ import annotations

import os
import sys

import numpy as np

from . import capi
from .search import SearchConfig, SearchResult, Searcher
from .workspace import Store, Workspace, WorkspaceConfig, _rust_lines, read_to_string, search_with_workspace


# ------------------------------------------------------------------ Rust formatting ------
def rust_display_f64(x: float) -> str:
    """`{}` of an f64: shortest digits that round-trip, positional, "1" for 1.0."""
    if x != x:
        return "NaN"
    if x in (float("inf"), float("-inf")):
        return "inf" if x > 0 else "-inf"
    return np.format_float_positional(np.float64(x), unique=True, trim="-")


def rust_display_f32(x: float) -> str:
    x = np.float32(x)
    if x != x:
        return "NaN"
    if np.isinf(x):
        return "inf" if x > 0 else "-inf"
    return np.format_float_positional(x, unique=True, trim="-")


def _json_f64(x: float) -> str:
    """serde_json (ryu): shortest round-trip; positional for 1e-5 <= |x| < 1e16 (ryu: -5 < kk <= 16) with a
    trailing ".0" on integral values; exponent form `1e-7` / `1.5e16` outside."""
    if x != x or x in (float("inf"), float("-inf")):
        return "null"                                     # serde_json writes non-finite floats as null
    if x == 0:
        return "-0.0" if str(x).startswith("-") else "0.0"
    a = abs(x)
    if 1e-5 <= a < 1e16:
        s = np.format_float_positional(np.float64(x), unique=True, trim="-")
        return s if "." in s else s + ".0"
    m, e = np.format_float_scientific(np.float64(x), unique=True, trim="-").split("e")
    return f"{m}e{int(e)}"


def _json_str(s: str) -> str:
    out = ['"']
    for ch in s:
        o = ord(ch)
        if ch == '"': out.append('\\"')
        elif ch == "\\": out.append("\\\\")
        elif ch == "\n": out.append("\\n")
        elif ch == "\r": out.append("\\r")
        elif ch == "\t": out.append("\\t")
        elif o == 8: out.append("\\b")
        elif o == 12: out.append("\\f")
        elif o < 0x20: out.append(f"\\u{o:04x}")
        else: out.append(ch)
    out.append('"')
    return "".join(out)


def to_string_pretty(value, indent: int = 0) -> str:
    """serde_json::to_string_pretty for dict (struct field order) / list / str / int / float."""
    pad, pad2 = "  " * indent, "  " * (indent + 1)
    if isinstance(value, dict):
        if not value:
            return "{}"
        items = [f"{pad2}{_json_str(k)}: {to_string_pretty(v, indent + 1)}" for k, v in value.items()]
        return "{\n" + ",\n".join(items) + "\n" + pad + "}"
    if isinstance(value, (list, tuple)):
        if not value:
            return "[]"
        return "[\n" + ",\n".join(pad2 + to_string_pretty(v, indent + 1) for v in value) + "\n" + pad + "]"
    if isinstance(value, bool):
        return "true" if value else "false"
    if isinstance(value, int):
        return str(value)
    if isinstance(value, float):
        return _json_f64(value)
    if value is None:
        return "null"
    return _json_str(str(value))


# ------------------------------------------------------------------ json_mode.rs ----------
def search_result_to_json(r: SearchResult) -> dict:          # cmds/search.rs:23-32
    return {"filename": r.filename, "start_line_number": r.start, "end_line_number": r.end,
            "match_line_number": r.match_line, "distance": float(r.distance), "content": "\n".join(r.lines)}


# ------------------------------------------------------------------ rendering -------------
def format_search_results(results, is_tty: bool) -> str:      # cmds/search.rs:35-63
    out = []
    for r in results:
        out.append(f"{r.filename}:{r.start}::{r.end} ({rust_display_f64(r.distance)})\n")
        for i, line in enumerate(r.lines):
            n = r.start + i
            if n == r.match_line and is_tty:
                out.append(f"\x1b[43m\x1b[30m{n + 1:4}: {line}\x1b[0m\n")
            else:
                out.append(f"{n + 1:4}: {line}\n")
        out.append("\n")
    return "".join(out)


def _read_lines(path):
    try:
        return _rust_lines(read_to_string(path))
    except (OSError, UnicodeDecodeError):
        return None


def format_workspace_search_results(ranked_lines, n_lines: int, is_tty: bool) -> str:   # cmds/search.rs:66-110
    out = []
    for rl in ranked_lines:
        m = rl.line_number
        start = max(0, m - n_lines)
        end = m + n_lines + 1                                 # NOT clamped in the header (:77-79)
        out.append(f"{rl.path}:{start}::{end} ({rust_display_f32(rl.distance)})\n")
        lines = _read_lines(rl.path)
        if lines is not None:
            actual_end = min(end, len(lines))
            if start > actual_end:
                raise IndexError("slice index starts past the end (the reference panics here)")
            for i, line in enumerate(lines[start:actual_end]):
                n = start + i
                if n == m and is_tty:
                    out.append(f"\x1b[43m\x1b[30m{n + 1:4}: {line}\x1b[0m\n")
                else:
                    out.append(f"{n + 1:4}: {line}\n")
        else:
            out.append("    [Error: Could not read file content]\n")
        out.append("\n")
    return "".join(out)


def workspace_results_to_json(ranked_lines, n_lines: int) -> list:   # cmds/search.rs:208-237
    res = []
    for rl in ranked_lines:
        m = rl.line_number
        start, end = max(0, m - n_lines), m + n_lines + 1
        lines = _read_lines(rl.path)
        content = "\n".join(lines[start:min(end, len(lines))]) if lines is not None \
            else "[Error: Could not read file content]"
        res.append({"filename": rl.path, "start_line_number": start, "end_line_number": end,
                    "match_line_number": m, "distance": float(np.float32(rl.distance)), "content": content})
    return res


# ------------------------------------------------------------------ search/mod.rs:49-75,122-143 ---
def create_document_from_content(searcher: Searcher, filename: str, content: str, model, ignore_case: bool):
    lines = _rust_lines(content)
    if not lines:
        return None                                            # :57-59
    emb_lines = [l.lower() for l in lines] if ignore_case else lines
    return searcher.add_document_lines(filename, lines, model, emb_lines)   # encode_with_args(.., Some(2048), 16384)


def search_files(files, query: str, model, config: SearchConfig, ctx: capi.Context | None = None):
    if model.ctx is None:
        model.ctx = ctx or capi.Context(0)
    searcher = Searcher(model.ctx, capi.Corpus(model.ctx, 1024))
    for f in files:
        content = read_to_string(f)                             # read_to_string(f)? -> error propagates
        create_document_from_content(searcher, f, content, model, config.ignore_case)
    q = model.encode_single(query)
    return searcher.search_documents(q, config)


# ------------------------------------------------------------------ cmds/search.rs:113-276 --
def search_cmd(query, files, n_lines, top_k, max_distance, ignore_case, json, workspace_name, model,
               stdin_lines=None, stdin_is_tty=True, stdout_is_tty=False, out=sys.stdout, err=sys.stderr) -> int:
    if ignore_case:
        query = query.lower()
    cfg = SearchConfig(n_lines, top_k, max_distance, ignore_case)
    if not files and not stdin_is_tty:
        lines = list(stdin_lines or [])
        if lines:
            if model.ctx is None:
                model.ctx = capi.Context(0)
            searcher = Searcher(model.ctx, capi.Corpus(model.ctx, 1024))
            emb = [l.lower() for l in lines] if ignore_case else lines
            searcher.add_document_lines("<stdin>", lines, model, emb)
            results = searcher.search_documents(model.encode_single(query), cfg)
            out.write(to_string_pretty({"results": [search_result_to_json(r) for r in results]}) + "\n" if json
                      else format_search_results(results, stdout_is_tty))
            return 0
    if not files:
        msg = "No input provided. Either specify files as arguments or pipe input to stdin."
        err.write(to_string_pretty({"error": msg, "error_type": "NoInput"}) + "\n" if json else f"Error: {msg}\n")
        return 1
    try:
        Workspace.active(workspace_name)
        in_ws = True
    except RuntimeError:
        in_ws = False
    if in_ws:
        if model.ctx is None:
            model.ctx = capi.Context(0)
        q = model.encode_single(query)
        ranked = search_with_workspace(files, q, lambda ls: model.encode_with_args(ls, 2048, 16384), cfg,
                                       workspace_name, ctx=model.ctx, log=lambda m: err.write(m + "\n"),
                                       model_fingerprint=model.fingerprint() if hasattr(model, "fingerprint") else None)
        out.write(to_string_pretty({"results": workspace_results_to_json(ranked, n_lines)}) + "\n" if json
                  else format_workspace_search_results(ranked, n_lines, stdout_is_tty))
    else:
        results = search_files(files, query, model, cfg)
        out.write(to_string_pretty({"results": [search_result_to_json(r) for r in results]}) + "\n" if json
                  else format_search_results(results, stdout_is_tty))
    return 0


# ------------------------------------------------------------------ cmds/workspace.rs ---------
def workspace_use_cmd(name: str, json: bool, out=sys.stdout) -> int:              # :11-67
    ws = Workspace(WorkspaceConfig(name=name, root_dir=Workspace.root_path(name)))
    ws.save()
    if json:
        try:
            total = Store.open(ws.config.root_dir).get_stats().total_documents
        except Exception:
            total = 0
        out.write(to_string_pretty({"name": ws.config.name, "root_dir": ws.config.root_dir, "total_documents": total}) + "\n")
    else:
        out.write(f"Workspace '{name}' configured.\nTo activate it, run:\n  export SEMTOOLS_WORKSPACE={name}\n\n"
                  "Or add this to your shell profile (.bashrc, .zshrc, etc.)\n\n"
                  "Or use the `--workspace` option on the commands that support it\n")
    return 0


def workspace_status_cmd(json: bool, workspace_name=None, out=sys.stdout) -> int:   # :69-113
    Workspace.active(workspace_name)
    ws = Workspace.open(workspace_name)
    stats = Store.open(ws.config.root_dir).get_stats()
    if json:
        out.write(to_string_pretty({"name": ws.config.name, "root_dir": ws.config.root_dir,
                                    "total_documents": stats.total_documents}) + "\n")
    else:
        out.write(f"Active workspace: {ws.config.name}\nRoot: {ws.config.root_dir}\nDocuments: {stats.total_documents}\n")
        out.write(f"Index: Yes ({stats.index_type or 'Unknown'})\n" if stats.has_index else "Index: No\n")
    return 0


def workspace_prune_cmd(json: bool, workspace_name=None, out=sys.stdout) -> int:    # :115-176
    Workspace.active(workspace_name)
    ws = Workspace.open(workspace_name)
    store = Store.open(ws.config.root_dir)
    all_paths = store.get_all_document_paths()
    missing = [p for p in all_paths if not os.path.exists(p)]
    if missing:
        store.delete_documents(missing)
    if json:
        out.write(to_string_pretty({"files_removed": len(missing), "files_remaining": len(all_paths) - len(missing)}) + "\n")
    elif not missing:
        out.write("No stale documents found. Workspace is clean.\n")
    else:
        out.write(f"Found {len(missing)} stale documents:\n" + "".join(f"  - {p}\n" for p in missing)
                  + f"Removed {len(missing)} stale documents from workspace.\n")
    return 0
