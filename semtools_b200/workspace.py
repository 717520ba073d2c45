"""Workspace embedding store -- the semantic contract of the reference's
src/workspace/mod.rs (Workspace, WorkspaceConfig) and src/workspace/store.rs (Store)
on a flat, GPU-friendly on-disk format.

The reference persists line vectors in two Qdrant Edge shards
(`documents.qdrant/`, `line_embeddings.qdrant/`, store.rs:113-183).  That segment /
WAL byte format is third-party and opaque, so BYTE compatibility with existing
`*.qdrant` directories is NOT provided (parity unpinned; SURVEY 8f-1).  What is kept,
name for name:

  Workspace.open / save / active / active_path / root_path       mod.rs:32-101
  WorkspaceConfig {name, root_dir, in_batch_size, oversample_factor}  mod.rs:8-25
  DocMeta {path,size_bytes,mtime,_version}, id = fnv1a(path)     store.rs:52-58,75-80
  LineEmbedding {path,line_number,embedding}, id = fnv1a(path||i32 LE)  :67-73,82-89
  Store.open / get_existing_docs / analyze_document_states / upsert_line_embeddings /
        upsert_document_metadata / search_line_embeddings / delete_documents /
        delete_document_metadata / delete_line_embeddings / get_all_document_paths /
        get_stats / count_documents / count_line_embeddings      store.rs:111-648
  CURRENT_EMBEDDING_VERSION = 2, LINE_EMBEDDING_SIZE = 256       store.rs:34,37

On disk (`<root_dir>/flat.b200/`):
  line_embeddings.f32   row-major N x 256 f32 -- exactly the HBM corpus matrix, so
                        opening a workspace is one read + one cudaMemcpy into a shard
  rows.i32              N x 2 int32: (path index, line_number) per row
  store.json            {"format", "paths": [...], "docs": [DocMeta...]}
Upserts overwrite the row whose id already exists and append otherwise, which
reproduces the reference's behaviour that rows of a shrunken file are NOT removed
(store.rs upsert only overwrites existing ids; SURVEY 3.3).

The nearest-neighbour query runs on the GPU (stb_search with row ranges = the path
filter, STB_MODE_STORE_QUERY); nothing here computes a distance on the CPU.
"""
from __future__ import annotations

import contextlib
import fcntl
import json
import os
from dataclasses import asdict, dataclass, field

import numpy as np

from . import capi
from .search import RankedLine

CURRENT_EMBEDDING_VERSION = 2     # store.rs:34
LINE_EMBEDDING_SIZE = 256         # store.rs:37
FORMAT = "semtools_b200.flat.v1"


# ------------------------------------------------------------------ mod.rs ------------
@dataclass
class WorkspaceConfig:
    """mod.rs:8-25 (in_batch_size / oversample_factor are unused vestiges upstream too)."""
    name: str = "default"
    root_dir: str = ""
    in_batch_size: int = 5_000
    oversample_factor: int = 3


def _home() -> str:
    home = os.environ.get("HOME") or os.path.expanduser("~")
    if not home:
        raise RuntimeError("No home dir found?")          # mod.rs:83
    return home


@dataclass
class Workspace:
    config: WorkspaceConfig

    @staticmethod
    def root_path(name: str) -> str:                       # mod.rs:82-91
        return os.path.join(_home(), ".semtools", "workspaces", name)

    @staticmethod
    def _config_path_for(name: str) -> str:                # mod.rs:93-101
        return os.path.join(_home(), ".semtools", "workspaces", name, "config.json")

    @staticmethod
    def active(workspace_name: str | None = None) -> str:  # mod.rs:69-79
        active = os.environ.get("SEMTOOLS_WORKSPACE", "") if workspace_name is None else workspace_name
        if not active:
            raise RuntimeError("No active workspace. Run: workspace use <name>")
        return active

    @staticmethod
    def active_path(workspace_name: str | None = None) -> str:   # mod.rs:58-67
        return Workspace.root_path(Workspace.active(workspace_name))

    @classmethod
    def open(cls, workspace_name: str | None = None) -> "Workspace":   # mod.rs:32-47
        active = cls.active(workspace_name)
        cfg = None
        try:
            with open(cls._config_path_for(active)) as f:
                d = json.load(f)
            cfg = WorkspaceConfig(**{k: d[k] for k in ("name", "root_dir", "in_batch_size", "oversample_factor")})
        except (OSError, ValueError, KeyError, TypeError):
            cfg = None
        config = cfg or WorkspaceConfig()
        if not config.root_dir:
            config.root_dir = cls.root_path(active)
        if not config.name or config.name == "default":
            config.name = active
        return cls(config)

    def save(self) -> None:                                # mod.rs:49-56
        p = self._config_path_for(self.config.name)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, "w") as f:
            json.dump(asdict(self.config), f, indent=2)    # serde_json::to_string_pretty


# ------------------------------------------------------------------ store.rs ----------
@dataclass
class DocMeta:
    path: str
    size_bytes: int
    mtime: int
    _version: int = CURRENT_EMBEDDING_VERSION

    def id(self) -> int:
        return capi.fnv1a64(self.path.encode("utf-8"))


@dataclass
class LineEmbedding:
    path: str
    line_number: int
    embedding: np.ndarray = field(repr=False, default=None)

    def id(self) -> int:
        return capi.line_id(self.path, self.line_number)


@dataclass
class DocumentInfo:                                        # search/mod.rs:26-30
    filename: str
    content: str
    meta: DocMeta


@dataclass
class DocumentState:                                       # store.rs:60-65
    kind: str                  # "Unchanged" | "Changed" | "New"
    filename: str
    info: DocumentInfo | None = None


@dataclass
class WorkspaceStats:                                      # store.rs:98-103
    total_documents: int
    has_index: bool
    index_type: str | None


class Store:
    """Flat-file restatement of store.rs `Store`."""

    def __init__(self, workspace_dir: str, ctx: capi.Context | None = None, _keep=None):
        self.dir = os.path.join(workspace_dir, "flat.b200")
        self.ctx = ctx
        self.model_fingerprint = getattr(_keep, "model_fingerprint", None)
        self.stored_model_fingerprint = None
        self._lock_depth = getattr(_keep, "_lock_depth", 0)
        self._gen = 0
        self._files = {"rows": "rows.i32", "emb": "line_embeddings.f32"}
        self._trailing = False
        self._paths: list = []                 # path table
        self._path_idx: dict = {}
        self._docs: dict = {}                  # path -> DocMeta
        self._rows = np.zeros((0, 2), dtype=np.int32)          # (path idx, line_number)
        self._emb = np.zeros((0, LINE_EMBEDDING_SIZE), dtype=np.float32)
        self._id_row: dict = {}                # LineEmbedding id -> row
        self._corpus = None                    # capi.Corpus mirror of self._emb (lazy)
        self._corpus_n = 0                     # rows of self._emb already uploaded to it
        # persistence bookkeeping: rows [0, _n_disk) are on disk and equal to memory except
        # _dirty_rows; _rewrite forces a full rewrite (first flush, deletions)
        self._n_disk = 0
        self._dirty_rows: set = set()
        self._rewrite = True
        self.full_rewrites = getattr(_keep, "full_rewrites", 0)   # how many flushes rewrote the row files (tests, diagnostics)

    # -- Store::open, store.rs:113-183 (creates the directories on first use)
    @classmethod
    def open(cls, workspace_dir: str, ctx: capi.Context | None = None, model_fingerprint: str | None = None) -> "Store":
        s = cls(workspace_dir, ctx)
        s.model_fingerprint = model_fingerprint
        os.makedirs(s.dir, exist_ok=True)
        with s._locked(exclusive=False):
            s._load()
        return s

    # Consistency protocol (shared with the C++ host, semtools_store.cpp):
    #  * store.json is the commit record: {"rows": committed row count, "gen": generation,
    #    "files": the two row files of this generation, "model": fingerprint of the embedder}.  It is
    #    replaced atomically (write tmp + rename) AFTER the row files hold the new state.
    #  * appends / in-place patches go to the current row files; rows beyond the committed count
    #    are garbage from an interrupted flush and are ignored on open (truncated by the next flush).
    #    A patched row whose commit never happened belongs to a document whose DocMeta is still the
    #    old one, so the next analyze_document_states sees it as Changed and re-embeds it.
    #  * anything that moves rows (deletions) writes NEW files (rows.<gen>.i32, ...) and commits
    #    by naming them in store.json; the old generation is unlinked afterwards.
    #  * flock(<dir>/.lock): shared while loading, exclusive around every mutation.  A mutation first
    #    checks the on-disk generation and reloads when another process committed in between, then
    #    applies itself to the fresh state -- nobody overwrites rows they never saw.
    @contextlib.contextmanager
    def _locked(self, exclusive: bool):
        if self._lock_depth:
            self._lock_depth += 1
            try:
                yield
            finally:
                self._lock_depth -= 1
            return
        fd = os.open(os.path.join(self.dir, ".lock"), os.O_RDWR | os.O_CREAT, 0o644)
        try:
            fcntl.flock(fd, fcntl.LOCK_EX if exclusive else fcntl.LOCK_SH)
            self._lock_depth = 1
            yield
        finally:
            self._lock_depth = 0
            try:
                fcntl.flock(fd, fcntl.LOCK_UN)
            finally:
                os.close(fd)

    def _disk_gen(self) -> int:
        try:
            with open(os.path.join(self.dir, "GEN")) as f:
                return int(f.read().strip() or 0)
        except (OSError, ValueError):
            return 0

    def _load(self) -> None:
        """(Re)load the committed state.  Caller holds the lock."""
        self.__init__(os.path.dirname(self.dir), self.ctx, _keep=self)
        meta_p = os.path.join(self.dir, "store.json")
        if not os.path.exists(meta_p):
            return
        with open(meta_p) as f:
            d = json.load(f)
        if d.get("format") != FORMAT:
            raise RuntimeError(f"unknown store format {d.get('format')!r}")
        try:                                     # a damaged commit record is a clear error, as in the C++ host
            self._paths = list(d["paths"])
            if not all(isinstance(p, str) for p in self._paths):
                raise TypeError("paths")
            self._path_idx = {p: i for i, p in enumerate(self._paths)}
            self._docs = {}
            for m in d["docs"]:
                dm = DocMeta(**m)
                if not isinstance(dm.path, str) or any(isinstance(v, bool) or not isinstance(v, int) for v in (dm.size_bytes, dm.mtime, dm._version)):
                    raise TypeError("docs")
                self._docs[dm.path] = dm
            self._gen = int(d.get("gen", 0))
            self._files = dict(d.get("files") or {"rows": "rows.i32", "emb": "line_embeddings.f32"})
            for key in ("rows", "emb"):
                name = self._files[key]
                if not isinstance(name, str) or not name or "/" in name or name.startswith("."):
                    raise ValueError("files")
            if "rows" in d and (isinstance(d["rows"], bool) or not isinstance(d["rows"], int) or d["rows"] < 0):
                raise ValueError("rows")
        except (KeyError, TypeError, ValueError, AttributeError) as e:
            raise RuntimeError(f"workspace store {self.dir}: store.json is corrupt ({e!r}); delete the directory to rebuild it") from e
        self.stored_model_fingerprint = d.get("model")
        rows_p, emb_p = os.path.join(self.dir, self._files["rows"]), os.path.join(self.dir, self._files["emb"])
        n_rows_file = os.path.getsize(rows_p) // 8 if os.path.exists(rows_p) else 0
        n_emb_file = os.path.getsize(emb_p) // (LINE_EMBEDDING_SIZE * 4) if os.path.exists(emb_p) else 0
        n = int(d["rows"]) if "rows" in d else min(n_rows_file, n_emb_file)
        if n_rows_file < n or n_emb_file < n:
            raise RuntimeError(f"workspace store {self.dir} is truncated: store.json commits {n} rows, the row files hold "
                               f"{n_rows_file} / {n_emb_file}; delete the directory to rebuild it")
        self._rows = np.fromfile(rows_p, dtype=np.int32, count=2 * n).reshape(-1, 2) if n else np.zeros((0, 2), dtype=np.int32)
        # copy-on-write map: a query-only process pages the matrix in once, straight into the
        # chunked GPU upload, instead of holding a second copy in RAM
        self._emb = np.memmap(emb_p, dtype=np.float32, mode="c", shape=(n, LINE_EMBEDDING_SIZE)) if n \
            else np.zeros((0, LINE_EMBEDDING_SIZE), dtype=np.float32)
        if n and (self._rows[:, 0].min() < 0 or self._rows[:, 0].max() >= len(self._paths)):
            raise RuntimeError(f"workspace store {self.dir} is corrupt: a row refers to path index "
                               f"{int(self._rows[:, 0].max())} but the path table has {len(self._paths)} entries; "
                               "delete the directory to rebuild it")
        if n:
            ids = capi.line_ids(self._paths, self._rows)                # one native call, not one per row
            self._id_row = {int(v): r for r, v in enumerate(ids)}
        self._n_disk, self._rewrite = n, False
        self._trailing = n_rows_file > n or n_emb_file > n              # garbage of an interrupted flush

    def _mutate(self, apply) -> None:
        """Run one mutation under the exclusive lock on a state that is current on disk, then commit."""
        with self._locked(exclusive=True):
            if self._disk_gen() != self._gen:
                self._load()                                             # another process committed since we loaded
            apply()
            self._flush()

    # -- flush_documents / flush_line_embeddings, store.rs:639-648
    def _flush(self) -> None:
        """store.json is rewritten every time (path table + DocMeta: small); the two row files
        are appended to / patched in place, and only rewritten (as a new generation) after deletions
        -- an upsert of a few files into a multi-GB store writes a few MB."""
        with self._locked(exclusive=True):
            gen = self._gen + 1
            files = dict(self._files)
            rows_p, emb_p = os.path.join(self.dir, files["rows"]), os.path.join(self.dir, files["emb"])
            n = len(self._rows)
            old_files = None
            if self._rewrite or not (os.path.exists(rows_p) and os.path.exists(emb_p)):
                if os.path.exists(rows_p) or os.path.exists(emb_p):      # never overwrite a committed generation in place
                    old_files = (rows_p, emb_p)
                    files = {"rows": f"rows.{gen}.i32", "emb": f"line_embeddings.{gen}.f32"}
                    rows_p, emb_p = os.path.join(self.dir, files["rows"]), os.path.join(self.dir, files["emb"])
                self._rows.astype(np.int32).tofile(rows_p)
                np.asarray(self._emb, dtype=np.float32).tofile(emb_p)
                self.full_rewrites += 1
            elif os.path.getsize(rows_p) < self._n_disk * 8 or os.path.getsize(emb_p) < self._n_disk * LINE_EMBEDDING_SIZE * 4:
                # the committed rows are no longer all there (foreign truncation): memory holds the full
                # state, so heal by writing a new generation instead of patching a damaged file
                old_files = (rows_p, emb_p)
                files = {"rows": f"rows.{gen}.i32", "emb": f"line_embeddings.{gen}.f32"}
                rows_p, emb_p = os.path.join(self.dir, files["rows"]), os.path.join(self.dir, files["emb"])
                self._rows.astype(np.int32).tofile(rows_p)
                np.asarray(self._emb, dtype=np.float32).tofile(emb_p)
                self.full_rewrites += 1
            else:
                with open(rows_p, "r+b") as fr, open(emb_p, "r+b") as fe:
                    # anything beyond the committed rows is the debris of an interrupted flush
                    fr.truncate(self._n_disk * 8); fe.truncate(self._n_disk * LINE_EMBEDDING_SIZE * 4)
                    for r in sorted(self._dirty_rows):
                        if r < self._n_disk:
                            fr.seek(r * 8); fr.write(self._rows[r].astype(np.int32).tobytes())
                            fe.seek(r * LINE_EMBEDDING_SIZE * 4); fe.write(np.asarray(self._emb[r], dtype=np.float32).tobytes())
                    if n > self._n_disk:
                        fr.seek(0, os.SEEK_END); fr.write(self._rows[self._n_disk:].astype(np.int32).tobytes())
                        fe.seek(0, os.SEEK_END); fe.write(np.asarray(self._emb[self._n_disk:], dtype=np.float32).tobytes())
                    fr.flush(); fe.flush()
                    os.fsync(fr.fileno()); os.fsync(fe.fileno())
            tmp = os.path.join(self.dir, "store.json.tmp")
            with open(tmp, "w") as f:
                json.dump({"format": FORMAT, "dim": LINE_EMBEDDING_SIZE, "rows": int(n), "gen": gen, "files": files,
                           "model": self.model_fingerprint or self.stored_model_fingerprint,
                           "paths": self._paths, "docs": [asdict(m) for m in self._docs.values()]}, f)
                f.flush(); os.fsync(f.fileno())
            os.replace(tmp, os.path.join(self.dir, "store.json"))        # the commit
            with open(os.path.join(self.dir, "GEN.tmp"), "w") as f:
                f.write(str(gen))
            os.replace(os.path.join(self.dir, "GEN.tmp"), os.path.join(self.dir, "GEN"))
            if old_files:
                for pth in old_files:
                    if os.path.exists(pth) and os.path.basename(pth) not in files.values():
                        os.unlink(pth)
            self._gen, self._files = gen, files
            self._n_disk, self._rewrite, self._trailing = n, False, False
            self._dirty_rows.clear()

    def flush_documents(self) -> None:
        self._flush()

    def flush_line_embeddings(self) -> None:
        self._flush()

    # -- store.rs:185-233
    def get_existing_docs(self, paths) -> dict:
        return {p: self._docs[p] for p in paths if p in self._docs}

    def _foreign_model(self) -> bool:
        """The store's vectors came from another embedder than this handle's (both known): every
        document counts as Changed, so it is re-embedded instead of being mixed in (no reference
        analogue -- the reference has one model; here two hosts with different tokenizers share a store)."""
        return bool(self.model_fingerprint and self.stored_model_fingerprint
                    and self.model_fingerprint != self.stored_model_fingerprint)

    # -- store.rs:549-611
    def analyze_document_states(self, file_paths) -> list:
        existing = self.get_existing_docs(file_paths)
        states = []
        for fp in file_paths:
            try:
                st = os.stat(fp)
            except OSError:
                continue                                             # :578-581 missing file: skipped
            cur = DocMeta(fp, st.st_size, int(st.st_mtime), CURRENT_EMBEDDING_VERSION)
            old = existing.get(fp)
            if old is not None and old.size_bytes == cur.size_bytes and old.mtime == cur.mtime \
                    and old._version == CURRENT_EMBEDDING_VERSION and not self._foreign_model():
                states.append(DocumentState("Unchanged", fp))
                continue
            content = read_to_string(fp)                             # invalid UTF-8 is an error
            states.append(DocumentState("Changed" if old is not None else "New", fp, DocumentInfo(fp, content, cur)))
        return states

    # -- store.rs:373-399
    def upsert_document_metadata(self, metas) -> None:
        if not metas:
            return

        def apply():
            for m in metas:
                self._docs[m.path] = m                               # same id (fnv1a(path)) -> replaced
        self._mutate(apply)

    # -- store.rs:402-434
    def upsert_line_embeddings(self, line_embeddings) -> None:
        if not line_embeddings:
            return
        self._mutate(lambda: self._apply_upsert_lines(line_embeddings))

    def _apply_upsert_lines(self, line_embeddings) -> None:
        new_rows, new_emb = [], []
        patched = {}                                                  # uploaded row -> its last vector of the batch
        for le in line_embeddings:
            emb = np.asarray(le.embedding, dtype=np.float32)
            if emb.shape != (LINE_EMBEDDING_SIZE,):
                raise ValueError("embedding must have 256 floats")
            pi = self._path_idx.get(le.path)
            if pi is None:
                pi = len(self._paths)
                self._paths.append(le.path)
                self._path_idx[le.path] = pi
            rid = le.id()
            row = self._id_row.get(rid)
            if row is not None and row < len(self._emb):
                self._emb[row] = emb                                  # upsert replaces by id
                self._rows[row] = (pi, le.line_number)
                self._dirty_rows.add(row)
                if row < self._corpus_n:
                    patched[row] = emb
            elif row is not None:                                     # replaced inside this same batch
                new_emb[row - len(self._emb)] = emb
            else:
                self._id_row[rid] = len(self._emb) + len(new_emb)
                new_rows.append((pi, le.line_number))
                new_emb.append(emb)
        if new_emb:
            self._emb = np.concatenate([self._emb, np.stack(new_emb)]) if len(self._emb) else np.stack(new_emb)
            self._rows = np.concatenate([self._rows, np.asarray(new_rows, dtype=np.int32).reshape(-1, 2)])
        # the GPU mirror takes in-place patches of its rows now; appended rows reach it lazily
        if patched and self._corpus is not None:
            idx = np.fromiter(sorted(patched), dtype=np.uint64, count=len(patched))
            self._mirror(lambda c: c.update(idx, np.stack([patched[int(r)] for r in idx])))

    def _mirror(self, change) -> None:
        """Apply one change to the GPU mirror; if the call fails the mirror is dropped and the next query
        uploads the rows again."""
        try:
            change(self._corpus)
        except capi.StbError:
            self._corpus = None

    # -- store.rs:235-296: only metadata of the CURRENT embedding version is deleted
    def delete_document_metadata(self, paths) -> None:
        def apply():
            for p in paths:
                m = self._docs.get(p)
                if m is not None and m._version == CURRENT_EMBEDDING_VERSION:
                    del self._docs[p]
        if paths:
            self._mutate(apply)

    # -- store.rs:298-357
    def delete_line_embeddings(self, paths) -> None:
        if not paths:
            return

        def apply():
            kill = {self._path_idx[p] for p in paths if p in self._path_idx}
            if kill:
                keep = ~np.isin(self._rows[:, 0], list(kill))
                if self._corpus is not None:                          # the mirror drops the same rows in place
                    gone = (~keep[: self._corpus_n]).astype(np.int8)
                    ranges = np.flatnonzero(np.diff(np.concatenate([[0], gone, [0]]))).reshape(-1, 2).astype(np.uint64)
                    if len(ranges):
                        self._mirror(lambda c: c.remove(ranges))
                        self._corpus_n -= int(gone.sum())
                self._rows = self._rows[keep]
                self._emb = np.ascontiguousarray(self._emb[keep])
                ids = capi.line_ids(self._paths, self._rows) if len(self._rows) else []
                self._id_row = {int(v): r for r, v in enumerate(ids)}
                self._rewrite = True                                  # rows moved: a new generation of row files
        self._mutate(apply)

    # -- store.rs:360-370
    def delete_documents(self, paths) -> None:
        if not paths:
            return
        self.delete_document_metadata(paths)
        self.delete_line_embeddings(paths)

    # -- store.rs:436-479
    def get_stats(self) -> WorkspaceStats:
        # the reference hard-codes "HNSW" (store.rs:440-444) although its shards use the
        # default plain index; this store really is an exact flat scan
        return WorkspaceStats(self.count_documents(), True, "FLAT")

    def get_all_document_paths(self) -> list:
        return [m.path for m in self._docs.values()]

    def count_documents(self) -> int:                                # store.rs:613-625
        return len(self._docs)

    def count_line_embeddings(self) -> int:                          # store.rs:627-637
        return int(len(self._emb))

    # -- GPU residency ---------------------------------------------------------------------
    def _gpu_corpus(self) -> capi.Corpus:
        if self.ctx is None:
            self.ctx = capi.Context(0)                               # no GPU -> StbError, never a CPU scan
        try:
            return self._upload_mirror(capi.Corpus)
        except capi.StbError as e:
            # The one rule for where the mirror lives: in HBM, unless creating or uploading it there fails with
            # STB_ERR_NOMEM; then its rows stay in host memory and only their q8 copy goes to HBM.  The hits are
            # the same either way.
            if e.status != capi.STB_ERR_NOMEM or (self._corpus is not None and self._corpus.host_rows):
                raise
            self._corpus = None
            return self._upload_mirror(capi.Corpus.in_host_memory)

    def _upload_mirror(self, make) -> capi.Corpus:
        if self._corpus is None:
            self._corpus = make(self.ctx, max(len(self._emb), 1))
            self._corpus_n = 0
        while self._corpus_n < len(self._emb):                        # only rows not uploaded yet, 256 MiB at a time
            hi = min(len(self._emb), self._corpus_n + 262144)
            self._corpus.append(self._emb[self._corpus_n:hi])
            self._corpus_n = hi
        return self._corpus

    def _ranges_for(self, subset_paths) -> np.ndarray:
        sel = [self._path_idx[p] for p in subset_paths if p in self._path_idx]
        if not sel or not len(self._rows):
            return np.zeros((0, 2), dtype=np.uint64)
        mask = np.isin(self._rows[:, 0], sel).astype(np.int8)
        edges = np.flatnonzero(np.diff(np.concatenate([[0], mask, [0]])))
        return edges.reshape(-1, 2).astype(np.uint64)

    # -- store.rs:481-546
    def search_line_embeddings(self, query_vec, subset_paths, top_k: int, max_distance=None) -> list:
        if len(subset_paths) == 0 or top_k == 0:                     # :489-491
            return []
        ranges = self._ranges_for(subset_paths)
        if len(ranges) == 0:
            return []
        hits = self._gpu_corpus().search(query_vec, top_k, max_distance, capi.STB_MODE_STORE_QUERY,
                                         row_ranges=ranges)
        return self._ranked(hits)

    def search_line_embeddings_batch(self, query_vecs, subset_paths, top_k: int, max_distance=None) -> list:
        """search_line_embeddings for many queries at once (stb_search_batch_filtered, one path filter for the
        batch): element i is what search_line_embeddings(query_vecs[i], subset_paths, top_k, max_distance)
        returns."""
        query_vecs = np.ascontiguousarray(query_vecs, dtype=np.float32).reshape(-1, capi.STB_DIM)
        if len(subset_paths) == 0 or top_k == 0:                     # :489-491
            return [[] for _ in range(len(query_vecs))]
        ranges = self._ranges_for(subset_paths)
        if len(ranges) == 0:
            return [[] for _ in range(len(query_vecs))]
        res = self._gpu_corpus().search_batch_filtered(query_vecs, ranges, top_k, max_distance)
        return [self._ranked(hits) for hits in res]

    def search_line_embeddings_many(self, query_vecs, subsets, top_k: int, max_distance=None) -> list:
        """search_line_embeddings for many queries, each with its own subset paths (stb_search_batch_subsets):
        element i is what search_line_embeddings(query_vecs[i], subsets[i], top_k, max_distance) returns."""
        query_vecs = np.ascontiguousarray(query_vecs, dtype=np.float32).reshape(-1, capi.STB_DIM)
        if len(subsets) != len(query_vecs):
            raise ValueError(f"{len(subsets)} subsets for {len(query_vecs)} queries")
        if top_k == 0 or len(query_vecs) == 0:                       # :489-491
            return [[] for _ in range(len(query_vecs))]
        # an empty subset, or one naming no stored path, has no ranges: 0 hits
        ranges = [self._ranges_for(paths) if len(paths) else np.zeros((0, 2), np.uint64) for paths in subsets]
        if not any(len(r) for r in ranges):
            return [[] for _ in range(len(query_vecs))]
        res = self._gpu_corpus().search_batch_subsets(query_vecs, ranges, top_k, max_distance)
        return [self._ranked(hits) for hits in res]

    def _ranked(self, hits) -> list:
        out = []
        for h in hits:
            pi, ln = self._rows[int(h["row"])]
            out.append(RankedLine(self._paths[pi], int(ln), float(np.float32(h["distance"]))))   # :531 f32
        return out


# ------------------------------------------------------------------ search/mod.rs:146-216 ---
def search_with_workspace(files, query_embedding, embed_lines, config, workspace_name=None, ctx=None,
                          log=None, model_fingerprint: str | None = None) -> list:
    """search_with_workspace: diff `files` against the store, embed only New/Changed
    documents (`embed_lines(list[str]) -> (n,256) f32`, i.e. create_document_from_content's
    encode_with_args on the caller's tokenizer + K3), upsert, then the filtered query."""
    ws = Workspace.open(workspace_name)
    store = Store.open(ws.config.root_dir, ctx, model_fingerprint=model_fingerprint)
    to_upsert, docs = [], []
    for st in store.analyze_document_states(files):
        if st.kind == "Unchanged":
            continue
        lines = _rust_lines(st.info.content)
        if not lines:
            continue                                                  # create_document_from_content -> None
        emb = embed_lines([l.lower() for l in lines] if config.ignore_case else lines)
        for i in range(len(lines)):
            to_upsert.append(LineEmbedding(st.filename, i, emb[i]))   # 0-based line numbers (:178)
        docs.append(st.info.meta)
    if to_upsert:
        if log:
            log(f"Updating workspace with {len(to_upsert)} lines from new/changed docs...")
        store.upsert_line_embeddings(to_upsert)
    if docs:
        if log:
            log(f"Updating workspace with {len(docs)} new/changed documents...")
        store.upsert_document_metadata(docs)
    max_d = None if config.max_distance is None else float(np.float32(config.max_distance))   # :211 `as f32`
    return store.search_line_embeddings(query_embedding, files, config.top_k, max_d)


def read_to_string(path: str) -> str:
    """fs::read_to_string: bytes decoded as UTF-8 (invalid UTF-8 is an error), NO newline
    translation -- Python's default text mode would turn a bare '\\r' into a line break, which
    str::lines() does not treat as one."""
    with open(path, encoding="utf-8", newline="") as f:
        return f.read()


def _rust_lines(content: str) -> list:
    """str::lines() (search/mod.rs:55): a line ends at '\\n'; a '\\r' directly before that
    '\\n' belongs to the terminator; no trailing empty line.  A bare '\\r' is ordinary text, and
    an unterminated last line keeps a trailing '\\r' (current Rust)."""
    if not content:
        return []
    parts = content.split("\n")
    last = parts.pop()                                   # text after the final '\n' (unterminated line)
    out = [p[:-1] if p.endswith("\r") else p for p in parts]
    if last != "":
        out.append(last)
    return out
