/**
 * GpuEmbeddingIndex — device-resident replacement for the `Map<string, number[]>` that
 * `VectorStore` keeps in RAM (src/knowledge/store/vector-store.ts:26), plus the one operation the
 * reference performs on it in its hot loop (:207-221): "all ids whose cosine with the query is
 * >= minScore, best first, stable, first 2*topK".
 *
 * NOT COMPILED in the build image (no Node/tsc); `compact()` below is no exception.  It is deliberately
 * tiny: the Map's ordered-key semantics (insertion slot, re-set keeps the slot, delete frees the key and
 * `compact()` later its slot) on top of the N-API addon (napi/rbk_napi.cc -> include/rbk_knn.h).  Searches take any
 * limit: bestBatch picks the one scan, the large-k search or the unbounded search by size.  The
 * tested mirror of the same bookkeeping is runbookai_b200/vector_store.py (`_set`, `delete_document`,
 * `_load_embeddings`, `compact`).
 * INTEGRATION.md shows the few lines of vector-store.ts that change to use it.
 */
// eslint-disable-next-line @typescript-eslint/no-var-requires
const { RbkIndex } = require('../native/build/Release/rbk_knn.node');

export interface ScoredId {
  id: string;
  score: number;
}

/** RUNBOOK_KNN_DEVICES="0,1,2,3" shards the corpus over those GPUs behind one handle (rbk_group_*). */
function devicesFromEnv(): number | number[] {
  const many = process.env.RUNBOOK_KNN_DEVICES;
  if (many) return many.split(',').map(Number);
  return Number(process.env.RUNBOOK_KNN_DEVICE ?? 0);
}

/**
 * RUNBOOK_KNN_F64_ON_HOST="1" keeps the float64 rows in pinned host memory instead of on the GPU (RBK_INDEX_F64_ON_HOST):
 * the same answers, about 5x the rows per GPU at d = 1536, host RAM and PCIe reads in the re-rank instead.
 */
function hostRowsFromEnv(): number {
  return process.env.RUNBOOK_KNN_F64_ON_HOST === '1' ? 1 : 0;
}

/**
 * RUNBOOK_KNN_SCAN_F16="1" makes the scan read per-row scaled fp16 rows instead of bf16 (RBK_INDEX_SCAN_F16): the same
 * answers and bytes per row, a tighter error bound, so fewer batches are rescanned with the wide candidate margin.
 */
function scanF16FromEnv(): number {
  return process.env.RUNBOOK_KNN_SCAN_F16 === '1' ? 1 : 0;
}

/**
 * RUNBOOK_KNN_EXACT_ROWS="f32" keeps the exact rows as float32 instead of float64 (RBK_INDEX_KEEP_F32): the same answers
 * at half the exact-row bytes while every embedding value is a float32.  "f32_split" (RBK_INDEX_KEEP_F32_SPLIT) halves
 * them again: the scan's bf16 copy holds each float32's high half, and only the low halves are kept beside it.  The addon reads the variable itself when its
 * constructor gets no `exactRows` argument, and widens the index to float64 in place (repeating the call) the first
 * time an append or overwrite holds a value no float32 can hold, so no embedding is ever refused.
 */
export type ExactRows = 'f64' | 'f32' | 'f32_split';

export class GpuEmbeddingIndex {
  private index: any | null = null;
  private idOfSlot: (string | null)[] = [];
  private slotOfId = new Map<string, number>();
  private dim = 0;
  /** ids whose stored vector has another length: while one is in the Map the reference's search throws (S2) */
  private badIds = new Set<string>();
  /** bestBatch calls between their device call and the slot -> id lookup; compact() waits for them */
  private inFlight = 0;
  private drained: Array<() => void> = [];
  /** set while compact() runs: new bestBatch calls wait for it */
  private compacting: Promise<void> | null = null;

  /**
   * One device index per resolved db path in the process, reference-counted: the reference builds and closes a
   * VectorStore per call site (hook-handlers.ts:329-337), which must not mean an upload per call.  `acquire`
   * returns the shared instance (first caller loads it), `release` frees the device memory with the last user.
   */
  private static shared = new Map<string, { ix: GpuEmbeddingIndex; refs: number; loaded: boolean }>();
  static acquire(dbPath: string): { ix: GpuEmbeddingIndex; needsLoad: boolean } {
    let e = GpuEmbeddingIndex.shared.get(dbPath);
    if (!e) {
      e = { ix: new GpuEmbeddingIndex(), refs: 0, loaded: false };
      GpuEmbeddingIndex.shared.set(dbPath, e);
    }
    e.refs++;
    const needsLoad = !e.loaded;
    e.loaded = true;
    return { ix: e.ix, needsLoad };
  }
  static release(dbPath: string): void {
    const e = GpuEmbeddingIndex.shared.get(dbPath);
    if (e && --e.refs === 0) {
      GpuEmbeddingIndex.shared.delete(dbPath);
      e.ix.index = null; // the addon's finalizer destroys the rbk_index / rbk_group
    }
  }

  constructor(private device: number | number[] = devicesFromEnv()) {}

  get size(): number {
    return this.slotOfId.size;
  }

  /** Bulk load at construction: rows are the f64-LE BLOBs exactly as SQLite returns them. */
  loadBlobs(rows: Array<{ id: string; embedding: Buffer }>): void {
    if (rows.length === 0) return;
    this.dim = rows[0].embedding.length / 8;
    const usable = rows.filter((r) => r.embedding.length === this.dim * 8);
    for (const r of rows) if (r.embedding.length !== this.dim * 8) this.badIds.add(r.id);
    this.index = new RbkIndex(this.dim, this.device, usable.length, hostRowsFromEnv(), scanF16FromEnv());
    // the Buffers go to the addon as they are: it packs them with memcpy and appends in one call
    const first = Number(this.index.appendBlobs(usable.map((r) => r.embedding)));
    usable.forEach((r, i) => this.remember(r.id, first + i));
  }

  /** Map.set: an existing key keeps its place in iteration order, a new key goes last. */
  set(id: string, embedding: number[]): void {
    if (!this.index) {
      this.dim = embedding.length;
      this.index = new RbkIndex(this.dim, this.device, 0, hostRowsFromEnv(), scanF16FromEnv());
    }
    const slot = this.slotOfId.get(id);
    if (embedding.length !== this.dim) {
      // the reference stores it and throws on every search until the id is deleted or re-set correctly
      this.badIds.add(id);
      if (slot !== undefined) {
        this.slotOfId.delete(id);
        this.idOfSlot[slot] = null;
        this.index.tombstone(BigInt64Array.from([BigInt(slot)]));
      }
      return;
    }
    this.badIds.delete(id);
    const row = Float64Array.from(embedding);
    if (slot !== undefined) this.index.overwriteF64(slot, row);
    else this.remember(id, Number(this.index.appendF64(row)));
  }

  /** addChunks: new ids are appended in one call, existing ids overwritten in one call (one host round trip each). */
  setMany(items: Array<{ id: string; embedding: number[] }>): void {
    const fresh = items.filter((it) => this.index && it.embedding.length === this.dim && !this.slotOfId.has(it.id));
    const again = items.filter((it) => this.index && it.embedding.length === this.dim && this.slotOfId.has(it.id));
    const rest = items.filter((it) => !fresh.includes(it) && !again.includes(it));
    if (new Set(items.map((it) => it.id)).size !== items.length) return items.forEach((it) => this.set(it.id, it.embedding));
    if (fresh.length > 0) {
      const packed = new Float64Array(fresh.length * this.dim);
      fresh.forEach((it, i) => packed.set(it.embedding, i * this.dim));
      const first = Number(this.index.appendF64(packed));
      fresh.forEach((it, i) => this.remember(it.id, first + i));
    }
    if (again.length > 0) {
      const packed = new Float64Array(again.length * this.dim);
      again.forEach((it, i) => packed.set(it.embedding, i * this.dim));
      this.index.overwriteF64Batch(BigInt64Array.from(again.map((it) => BigInt(this.slotOfId.get(it.id)!))), packed);
      again.forEach((it) => this.badIds.delete(it.id));
    }
    rest.forEach((it) => this.set(it.id, it.embedding));
  }

  /** Map.delete for a batch of keys. */
  deleteMany(ids: string[]): void {
    const slots: bigint[] = [];
    for (const id of ids) {
      this.badIds.delete(id);
      const slot = this.slotOfId.get(id);
      if (slot === undefined) continue;
      this.slotOfId.delete(id);
      this.idOfSlot[slot] = null;
      slots.push(BigInt(slot));
    }
    if (slots.length > 0 && this.index) this.index.tombstone(BigInt64Array.from(slots));
  }

  clear(): void {
    this.idOfSlot = [];
    this.slotOfId.clear();
    this.badIds.clear();
    this.index?.clear();
  }

  /** The scan + threshold + stable sort + cut, for one query embedding. */
  async best(query: number[], limit: number, minScore: number): Promise<ScoredId[]> {
    return (await this.bestBatch([query], limit, minScore))[0];
  }

  /**
   * The same for B queries in ONE device pass (what B sequential search() calls cost the reference): the entry point
   * of the micro-batcher that coalesces concurrent searches of several investigations (SURVEY 8f-3;
   * runbookai_b200/batcher.py is the tested mirror).  limit <= 112 takes one scan (RBK_MAX_K_FETCH); up to 4096
   * (RBK_MAX_K_FETCH_LARGE) the large-k search (two scans and an exact re-rank); any larger limit the unbounded search
   * (the same two scans, the candidates sorted on the GPU), so every topK the reference accepts is answered.
   */
  async bestBatch(queries: number[][], limit: number, minScore: number): Promise<ScoredId[][]> {
    while (this.compacting) await this.compacting; // never search against a table that is being renumbered
    if (!this.index || this.slotOfId.size === 0) return queries.map(() => []);
    if (this.badIds.size > 0 || queries.some((q) => q.length !== this.dim)) {
      throw new Error('Vectors must have the same length');
    }
    const B = queries.length;
    const packed = new Float64Array(B * this.dim);
    queries.forEach((q, b) => packed.set(q, b * this.dim));
    this.inFlight++;
    try {
      const { slots, scores, counts } =
        limit > 4096
          ? await this.index.searchUnbounded(packed, B, limit, minScore)
          : limit > 112
            ? await this.index.searchLarge(packed, B, limit, minScore)
            : await this.index.search(packed, B, limit, minScore);
      return queries.map((_, b) => {
        const out: ScoredId[] = [];
        for (let i = 0; i < counts[b]; i++) {
          out.push({ id: this.idOfSlot[Number(slots[b * limit + i])]!, score: scores[b * limit + i] });
        }
        return out;
      });
    } finally {
      if (--this.inFlight === 0) this.drained.splice(0).forEach((wake) => wake());
    }
  }

  /** Whether bestEach is available: the loaded addon's library has the per-query search (rbk_*_search_each_f64). */
  get hasBestEach(): boolean {
    return this.index !== null && this.index.hasSearchEach === true;
  }

  /**
   * bestBatch with each query at its own limit and minScore, in ONE native call (rbk_*_search_each_f64): one scan when
   * every limit is <= 112, else the two scans of the large-k search for all of them.  Result b is exactly what
   * best(queries[b], limits[b], minScores[b]) returns.  Throws against a library without the per-query search
   * (hasBestEach false).
   */
  async bestEach(queries: number[][], limits: number[], minScores: number[]): Promise<ScoredId[][]> {
    while (this.compacting) await this.compacting; // never search against a table that is being renumbered
    if (!this.index || this.slotOfId.size === 0) return queries.map(() => []);
    if (this.badIds.size > 0 || queries.some((q) => q.length !== this.dim)) {
      throw new Error('Vectors must have the same length');
    }
    const B = queries.length;
    const packed = new Float64Array(B * this.dim);
    queries.forEach((q, b) => packed.set(q, b * this.dim));
    const K = Math.max(1, ...limits);
    this.inFlight++;
    try {
      const { slots, scores, counts } = await this.index.searchEach(
        packed, B, Int32Array.from(limits), Float64Array.from(minScores));
      return queries.map((_, b) => {
        const out: ScoredId[] = [];
        for (let i = 0; i < counts[b]; i++) {
          out.push({ id: this.idOfSlot[Number(slots[b * K + i])]!, score: scores[b * K + i] });
        }
        return out;
      });
    } finally {
      if (--this.inFlight === 0) this.drained.splice(0).forEach((wake) => wake());
    }
  }

  /** Whether mmrEach is available: the loaded addon's library has the MMR search (rbk_*_search_mmr_f64). */
  get hasMmrEach(): boolean {
    return this.index !== null && this.index.hasSearchMmr === true;
  }

  /**
   * Diverse hits by maximal marginal relevance, in ONE native call (rbk_*_search_mmr_f64): query b's limits[b] picks
   * from the fetchKs[b] hits bestEach would return at minScores[b], each the candidate whose lambdas[b] * score -
   * (1 - lambdas[b]) * (largest cosine to a pick so far) is largest, in selection order with their scores.  Throws for a
   * limit < 1, a fetchK below its limit or above 4096, or a lambda outside [0, 1] (the library's checks), and against a
   * library without the MMR search (hasMmrEach false).
   */
  async mmrEach(queries: number[][], limits: number[], fetchKs: number[], lambdas: number[],
                minScores: number[]): Promise<ScoredId[][]> {
    while (this.compacting) await this.compacting; // never search against a table that is being renumbered
    if (!this.index || this.slotOfId.size === 0) return queries.map(() => []);
    if (this.badIds.size > 0 || queries.some((q) => q.length !== this.dim)) {
      throw new Error('Vectors must have the same length');
    }
    const B = queries.length;
    const packed = new Float64Array(B * this.dim);
    queries.forEach((q, b) => packed.set(q, b * this.dim));
    const K = Math.max(0, ...limits);
    this.inFlight++;
    try {
      const { slots, scores, counts } = await this.index.searchMmr(packed, B, Int32Array.from(limits),
        Int32Array.from(fetchKs), Float64Array.from(lambdas), Float64Array.from(minScores));
      return queries.map((_, b) => {
        const out: ScoredId[] = [];
        for (let i = 0; i < counts[b]; i++) {
          out.push({ id: this.idOfSlot[Number(slots[b * K + i])]!, score: scores[b * K + i] });
        }
        return out;
      });
    } finally {
      if (--this.inFlight === 0) this.drained.splice(0).forEach((wake) => wake());
    }
  }

  /** Whether similarEach is available: the loaded addon's library has search by slot (rbk_*_search_slots_f64). */
  get hasSimilarEach(): boolean {
    return this.index !== null && this.index.hasSearchSlots === true;
  }

  /**
   * bestEach whose queries are the stored embeddings of ids (the chunks most like a stored chunk), read where the index
   * keeps them: no embedding call.  Result b is exactly what best(embedding of ids[b], limits[b], minScores[b]) returns,
   * ids[b] itself included.  Throws for an id the Map does not hold, and against a library without search by slot
   * (hasSimilarEach false).
   */
  async similarEach(ids: string[], limits: number[], minScores: number[]): Promise<ScoredId[][]> {
    while (this.compacting) await this.compacting; // never search against a table that is being renumbered
    if (this.badIds.size > 0) throw new Error('Vectors must have the same length');
    const querySlots = ids.map((id) => {
      const slot = this.slotOfId.get(id);
      if (slot === undefined) throw new Error(`no embedding for id ${id}`);
      return BigInt(slot);
    });
    if (!this.index || ids.length === 0) return [];
    const K = Math.max(1, ...limits);
    this.inFlight++;
    try {
      const { slots, scores, counts } = await this.index.searchSlots(
        BigInt64Array.from(querySlots), ids.length, Int32Array.from(limits), Float64Array.from(minScores));
      return ids.map((_, b) => {
        const out: ScoredId[] = [];
        for (let i = 0; i < counts[b]; i++) {
          out.push({ id: this.idOfSlot[Number(slots[b * K + i])]!, score: scores[b * K + i] });
        }
        return out;
      });
    } finally {
      if (--this.inFlight === 0) this.drained.splice(0).forEach((wake) => wake());
    }
  }

  /** Whether similarPairs is available: the loaded addon's library has rbk_*_similar_pairs_f64. */
  get hasSimilarPairs(): boolean {
    return this.index !== null && this.index.hasSimilarPairs === true;
  }

  /**
   * Every pair of stored embeddings whose cosine is >= minScore ("which chunks are near-duplicates of each other"),
   * exactly, each pair once: [idA, idB, score] in the engine's order (idA's slot ascending, then score descending, ties
   * by idB's slot ascending).  The addon answers in pages of whole rows; this loops them until the pass is complete.
   * Throws on a ragged Map (as best does) and against a library without similar pairs (hasSimilarPairs false).
   */
  async similarPairs(minScore: number): Promise<Array<[string, string, number]>> {
    while (this.compacting) await this.compacting; // never search against a table that is being renumbered
    if (this.badIds.size > 0) throw new Error('Vectors must have the same length');
    if (!this.index || this.slotOfId.size === 0) return [];
    const end = this.idOfSlot.length;
    const page = Math.max(end, 1 << 20);
    const out: Array<[string, string, number]> = [];
    this.inFlight++;
    try {
      for (let next = 0; next < end; ) {
        const { a, b, scores, nextSlot } = await this.index.similarPairs(minScore, next, page);
        for (let i = 0; i < scores.length; i++) {
          out.push([this.idOfSlot[Number(a[i])]!, this.idOfSlot[Number(b[i])]!, scores[i]]);
        }
        next = Number(nextSlot);
      }
      return out;
    } finally {
      if (--this.inFlight === 0) this.drained.splice(0).forEach((wake) => wake());
    }
  }

  /**
   * Give the slots of deleted ids back (the reference's Map.delete frees its entry; a tombstone alone does not): the
   * device index moves its live rows down in Map order and returns oldToNew, through which slotOfId and idOfSlot are
   * renumbered.  Holds back new bestBatch calls and waits for those in flight first, so no search result is ever mapped
   * through the other table.  Returns the number of slots reclaimed.  A device group (RUNBOOK_KNN_DEVICES) compacts
   * the same way, in global slots, moving rows between its GPUs; only a library built before group compaction throws.
   */
  async compact(): Promise<number> {
    while (this.compacting) await this.compacting;
    let done!: () => void;
    this.compacting = new Promise<void>((resolve) => (done = resolve));
    try {
      if (this.inFlight > 0) await new Promise<void>((resolve) => this.drained.push(resolve));
      if (!this.index) return 0;
      const oldToNew: BigInt64Array = this.index.compact();
      const ids: (string | null)[] = [];
      this.idOfSlot.forEach((id, slot) => {
        if (id === null || id === undefined) return;
        const to = Number(oldToNew[slot]);
        ids[to] = id;
        this.slotOfId.set(id, to);
      });
      this.idOfSlot = ids;
      return oldToNew.length - ids.length;
    } finally {
      this.compacting = null;
      done();
    }
  }

  /**
   * Give unused device memory back (after compact() or clear()): the capacity drops to what the rows need and the
   * scratch buffers are released.  No slot moves, so searches in flight need no waiting; the native call waits for
   * the index's queued device work itself.
   */
  trim(): void {
    this.index?.trim();
  }

  /**
   * Change the storage tier of the loaded index in place (rbk_index_set_tier / rbk_group_set_tier): `f64OnHost` moves
   * the float64 rows between the GPU and pinned host memory, `scanF16` switches the scan between bf16 and fp16.  An
   * omitted key keeps its setting; `exactRows` widens ('f64') or narrows ('f32' or 'f32_split', refused unless every
   * stored value is a float32) the exact rows.  Answers and slots do not change, so nothing is remapped; the native call waits
   * for the index's queued device work itself.  Nothing is automatic: an append that throws for lack of device memory
   * is the caller's to retry after `setTier({ f64OnHost: true })`.  Throws (with the index unchanged) if the new tier
   * cannot be backed, and against a library built before tier changes.
   */
  setTier(tier: { f64OnHost?: boolean; scanF16?: boolean; exactRows?: ExactRows }): void {
    this.index?.setTier(tier);
  }

  /** Where the exact rows live, which scan runs and the exact rows' width, as they are now; null before the first row
   * is loaded. */
  get tier(): { f64OnHost: boolean; scanF16: boolean; exactRows: ExactRows } | null {
    return this.index ? this.index.tier : null;
  }

  private remember(id: string, slot: number): void {
    this.slotOfId.set(id, slot);
    this.idOfSlot[slot] = id;
  }
}

/**
 * Query micro-batcher (SURVEY 8f-3): concurrent `best()` calls that arrive within `windowMs` share ONE device pass
 * and every caller gets exactly what its own `best()` would have returned.  With a library that has the per-query
 * search (`hasBestEach`) the window is ONE `bestEach` at every caller's own limit and minScore, callers above one
 * scan's limit (112) included; only a limit that is not an integer in [1, 4096] goes through on its own (its own error,
 * or a result that would make every row of the shared one that wide).  Without it the pass (`bestBatch`) fetches for
 * the most demanding caller (largest limit, lowest minScore), each caller's own `>= minScore` and cut are re-applied,
 * and callers above 112 go through on their own, to the large-k search.  runbookai_b200/batcher.py is the tested
 * mirror of this class (same coalescing, same per-caller answers, same behaviour on close).
 */
export class SearchBatcher {
  private queue: Array<{
    query: number[];
    limit: number;
    minScore: number;
    resolve: (r: ScoredId[]) => void;
    reject: (e: unknown) => void;
  }> = [];
  private timer: ReturnType<typeof setTimeout> | null = null;
  private closed = false;
  batches = 0;

  constructor(private index: GpuEmbeddingIndex, private windowMs = 2, private maxBatch = 256) {}

  best(query: number[], limit: number, minScore: number): Promise<ScoredId[]> {
    if (this.closed) return Promise.reject(new Error('batcher closed'));
    const alone = this.index.hasBestEach ? !(Number.isInteger(limit) && limit >= 1 && limit <= 4096) : limit > 112;
    if (alone) return this.index.best(query, limit, minScore);
    return new Promise((resolve, reject) => {
      this.queue.push({ query, limit, minScore, resolve, reject });
      if (this.queue.length >= this.maxBatch) this.flush();
      else if (!this.timer) this.timer = setTimeout(() => this.flush(), this.windowMs);
    });
  }

  close(): void {
    this.closed = true;
    if (this.timer) clearTimeout(this.timer);
    this.timer = null;
    for (const w of this.queue.splice(0)) w.reject(new Error('batcher closed'));
  }

  private flush(): void {
    if (this.timer) clearTimeout(this.timer);
    this.timer = null;
    const batch = this.queue.splice(0, this.maxBatch);
    if (batch.length === 0) return;
    if (this.queue.length > 0) this.timer = setTimeout(() => this.flush(), 0);
    this.batches++;
    if (this.index.hasBestEach) {
      this.index
        .bestEach(batch.map((w) => w.query), batch.map((w) => w.limit), batch.map((w) => w.minScore))
        .then((all) => batch.forEach((w, i) => w.resolve(all[i])))
        .catch((e) => batch.forEach((w) => w.reject(e)));
      return;
    }
    const limit = Math.max(...batch.map((w) => w.limit));
    const minScore = Math.min(...batch.map((w) => w.minScore));
    this.index
      .bestBatch(batch.map((w) => w.query), limit, minScore)
      .then((all) =>
        batch.forEach((w, i) => w.resolve(all[i].filter((h) => h.score >= w.minScore).slice(0, w.limit))),
      )
      .catch((e) => batch.forEach((w) => w.reject(e))); // every waiter gets the error its own best() would have thrown
  }
}

