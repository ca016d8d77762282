/**
 * napi/gpu-backend.ts -- the reference-side glue a maintainer of @vainplex/openclaw-governance would add
 * (packages/openclaw-governance/src/gpu-backend.ts).  It keeps the plugin's classes and call sites and swaps the two hot
 * loops and the hash for calls into the N-API addon built from napi/openclaw_gov_napi.c:
 *
 *   PatternRegistry.findMatches   src/redaction/registry.ts:212-242,288-316   -> findMatchesOne / findMatchesFew / findMatchesBatch (spans already resolved)
 *   matchesAny                    src/conditions/context.ts:9-25              -> scanBatch over every pattern of the policy set
 *   ResponseGate mustMatch / mustNotMatch  src/response-gate.ts:104-149       -> scanBatch
 *   tool param `matches`          src/conditions/tool.ts:36-45                -> scanBatch
 *   PolicyEvaluator.evaluate      src/policy-evaluator.ts:18-146              -> policyEvalOne (GpuPolicyEvaluator)
 *   sha256                        src/util.ts:77-79, src/redaction/vault.ts:26-28 -> sha256Batch
 *   audit JSONL -> Merkle log     src/audit-trail.ts:151-179 (flush)          -> logAppendJsonl / logRoot / logFrontier
 *
 * Not compiled or run in this repository (no Node.js in the image or on the GPU box): it documents the binding;
 * vainplex_openclaw_b200/plugin.py is the executable mirror of the same wiring and is what the tests drive.
 */
import { createRequire } from "node:module";

const require = createRequire(import.meta.url);

type Addon = {
  init(device?: number): void;
  shutdown(): void;
  stats(): Record<string, number>;
  ruleCheck(source: string, flags?: number): number;
  createRuleset(rules: { source: string; flags?: number; category?: number }[]): { handle: unknown; status: Int32Array };
  scanBatch(handle: unknown, bytes: Uint8Array, offsets: Uint32Array): { words: BigUint64Array; hits: Uint32Array };
  scanOne(handle: unknown, bytes: Uint8Array): { word: bigint; rules: Uint32Array };
  findMatchesBatch(handle: unknown, bytes: Uint8Array, offsets: Uint32Array): Uint32Array;
  redactBatch(handle: unknown, bytes: Uint8Array, offsets: Uint32Array): { bytes: Uint8Array; offsets: Uint32Array; spans: Uint32Array; digests: Uint8Array };
  findMatchesOne(handle: unknown, bytes: Uint8Array): Uint32Array;
  redactOne(handle: unknown, bytes: Uint8Array): { bytes: Uint8Array; spans: Uint32Array; digests: Uint8Array };
  // the strings of one scanned value, blocking, one device round trip (up to 256 strings and 64 KB): the batch calls' results
  findMatchesFew(handle: unknown, bytes: Uint8Array, offsets: Uint32Array): Uint32Array;
  redactFew(handle: unknown, bytes: Uint8Array, offsets: Uint32Array): { bytes: Uint8Array; offsets: Uint32Array; spans: Uint32Array; digests: Uint8Array };
  setPolicy(handle: unknown, rulePolicy: Uint32Array, ruleAction: Uint8Array): void;
  verdictBatch(handle: unknown, bytes: Uint8Array, offsets: Uint32Array): Uint32Array;
  // per-message views of one rule set: rows = nViews x ceil(nRules / 32) words (bit r = rule r in the view); views = one id
  // per message -- an exempt tool's output on the credential view, a context on the view of its in-scope policies
  setViews(handle: unknown, rows: Uint32Array, nViews: number): void;
  scanBatchViews(handle: unknown, bytes: Uint8Array, offsets: Uint32Array, views: Uint8Array): { words: BigUint64Array; hits: Uint32Array };
  findMatchesBatchViews(handle: unknown, bytes: Uint8Array, offsets: Uint32Array, views: Uint8Array): Uint32Array;
  redactBatchViews(handle: unknown, bytes: Uint8Array, offsets: Uint32Array, views: Uint8Array): { bytes: Uint8Array; offsets: Uint32Array; spans: Uint32Array; digests: Uint8Array };
  verdictBatchViews(handle: unknown, bytes: Uint8Array, offsets: Uint32Array, views: Uint8Array): Uint32Array;
  // whole policies on the device (openclaw_gov.h: program layout): one verdict per context, (ctx, program rule) match pairs
  setPolicyProgram(handle: unknown, program: Uint32Array, nAtoms: number): void;
  policyEvalBatch(handle: unknown, bytes: Uint8Array, offsets: Uint32Array, roles: Uint8Array, ctxOffsets: Uint32Array, atoms: Uint32Array,
                  nAtoms: number): { verdicts: Uint32Array; matches: Uint32Array };
  // one context owning every text, blocking, one device round trip: policyEvalBatch's verdict word and program rules for it
  policyEvalOne(handle: unknown, bytes: Uint8Array, offsets: Uint32Array, roles: Uint8Array, atoms: Uint32Array, nAtoms: number): { verdict: number; rules: Uint32Array };
  sha256Batch(bytes: Uint8Array, offsets: BigUint64Array): Uint8Array;
  merkleRoot(bytes: Uint8Array, offsets: BigUint64Array): Uint8Array;
  logCreate(keepLeafDigests: boolean): unknown;
  logRestore(size: bigint, frontier: Uint8Array): unknown;
  logAppendJsonl(log: unknown, bytes: Uint8Array): bigint;
  logRoot(log: unknown): Uint8Array;
  logSize(log: unknown): bigint;
  logFrontier(log: unknown): Uint8Array;
  logProof(log: unknown, index: bigint): Uint8Array;
  logConsistency(log: unknown, firstSize: bigint): Uint8Array;
  logCreateTree(): unknown;
  logProofs(log: unknown, indices: BigUint64Array, treeSize: bigint): { paths: Uint8Array; lens: Uint32Array };
  logConsistencyBetween(log: unknown, firstSize: bigint, secondSize: bigint): Uint8Array;
  verifyProofs(leafBytes: Uint8Array, leafOffsets: BigUint64Array, indices: BigUint64Array, treeSize: bigint, paths: Uint8Array,
               lens: Uint32Array, stride: number, root: Uint8Array): Uint8Array;
};

const addon: Addon = require("./openclaw_gov.node");
const FLAG_ICASE = 1;
const CATEGORY: Record<string, number> = { credential: 0, pii: 1, financial: 2, custom: 3 };
const enc = new TextEncoder();

/** Buffer.from(s, "utf8") for a batch: one byte array + offsets (what every batch entry point takes). */
export function pack(texts: string[]): { bytes: Uint8Array; offsets: Uint32Array } {
  const parts = texts.map((t) => enc.encode(t));
  const offsets = new Uint32Array(parts.length + 1);
  parts.forEach((p, i) => (offsets[i + 1] = offsets[i] + p.length));
  const bytes = new Uint8Array(offsets[parts.length] + 16);            // 16 bytes of slack: the device reads whole chunks
  parts.forEach((p, i) => bytes.set(p, offsets[i]));
  return { bytes, offsets };
}

export function initGpu(device?: number): void {
  addon.init(device);                                                  // throws without a usable H100: failMode decides (src/hooks.ts:232-241)
}

/** Drop-in for PatternRegistry (src/redaction/registry.ts:157-316): same constructor arguments, same findMatches result. */
export class GpuPatternRegistry {
  private readonly patterns: { id: string; category: string; regex: RegExp; replacementType: string }[];
  private readonly handle: unknown;

  constructor(patterns: { id: string; category: string; regex: RegExp; replacementType: string }[]) {
    const created = addon.createRuleset(
      patterns.map((p) => ({ source: p.regex.source, flags: p.regex.ignoreCase ? FLAG_ICASE : 0, category: CATEGORY[p.category] ?? 3 })),
    );
    // a pattern outside the supported subset never matches and is dropped, exactly like a failed compileCustomPattern (registry.ts:249-281)
    this.patterns = patterns.filter((_, i) => created.status[i] === 0);
    this.handle = addon.createRuleset(
      this.patterns.map((p) => ({ source: p.regex.source, flags: p.regex.ignoreCase ? FLAG_ICASE : 0, category: CATEGORY[p.category] ?? 3 })),
    ).handle;
  }

  /** findMatches for many strings at once; per string the same array PatternRegistry.findMatches returns. */
  findMatchesBatch(texts: string[]): { pattern: (typeof this.patterns)[number]; match: string; index: number; length: number }[][] {
    const { bytes, offsets } = pack(texts);
    const spans = addon.findMatchesBatch(this.handle, bytes, offsets);  // msg, rule, startByte, endByte, start16, end16 -- overlaps already resolved
    const out: ReturnType<GpuPatternRegistry["findMatchesBatch"]> = texts.map(() => []);
    for (let k = 0; k < spans.length; k += 6) {
      const [msg, rule, , , s16, e16] = spans.subarray(k, k + 6);
      out[msg].push({ pattern: this.patterns[rule], match: texts[msg].slice(s16, e16), index: s16, length: e16 - s16 });
    }
    return out;
  }

  /** findMatches for one string (the synchronous hooks' path): one blocking call, one device round trip. */
  findMatches(text: string): ReturnType<GpuPatternRegistry["findMatchesBatch"]>[number] {
    const spans = addon.findMatchesOne(this.handle, enc.encode(text));   // msg (= 0), rule, startByte, endByte, start16, end16
    const out: ReturnType<GpuPatternRegistry["findMatchesBatch"]>[number] = [];
    for (let k = 0; k < spans.length; k += 6) {
      const [, rule, , , s16, e16] = spans.subarray(k, k + 6);
      out.push({ pattern: this.patterns[rule], match: text.slice(s16, e16), index: s16, length: e16 - s16 });
    }
    return out;
  }

  /** findMatches for every string leaf of one value RedactionEngine.scanValue walks (src/redaction/engine.ts:94-147), collected
   *  in walk order: one blocking call, one device round trip; per string the same array findMatches returns. */
  findMatchesFew(texts: string[]): ReturnType<GpuPatternRegistry["findMatchesBatch"]> {
    const { bytes, offsets } = pack(texts);
    const spans = addon.findMatchesFew(this.handle, bytes, offsets);    // msg, rule, startByte, endByte, start16, end16
    const out: ReturnType<GpuPatternRegistry["findMatchesBatch"]> = texts.map(() => []);
    for (let k = 0; k < spans.length; k += 6) {
      const [msg, rule, , , s16, e16] = spans.subarray(k, k + 6);
      out[msg].push({ pattern: this.patterns[rule], match: texts[msg].slice(s16, e16), index: s16, length: e16 - s16 });
    }
    return out;
  }
}

/** matchesAny (src/conditions/context.ts:9-25) for a whole policy set: every pattern is one rule, one scan per batch of texts. */
export class GpuRuleScanner {
  private readonly handle: unknown;
  private readonly ruleOfPattern: number[] = [];

  constructor(rules: (string | string[])[]) {
    const srcs: { source: string }[] = [];
    rules.forEach((pats, ri) => {
      for (const p of Array.isArray(pats) ? pats : [pats]) {
        // context.ts:15-17: a pattern that is not a valid RegExp falls back to includes() -- compiled as an escaped literal
        const source = addon.ruleCheck(p) === -4 /* CG_ERR_SYNTAX */ ? p.replace(/[.*+?^${}()|[\]\\\/-]/g, "\\$&") : p;
        srcs.push({ source });
        this.ruleOfPattern.push(ri);
      }
    });
    this.handle = addon.createRuleset(srcs).handle;
  }

  /** -> per text the sorted rule indices with a matching pattern */
  scan(texts: string[]): number[][] {
    const { bytes, offsets } = pack(texts);
    const { hits } = addon.scanBatch(this.handle, bytes, offsets);
    const out: Set<number>[] = texts.map(() => new Set());
    for (let k = 0; k < hits.length; k += 2) out[hits[k]].add(this.ruleOfPattern[hits[k + 1]]);
    return out.map((s) => [...s].sort((a, b) => a - b));
  }
}

/** A policy list compiled for setPolicyProgram, as plugin.PolicyEvaluator._compile_program compiles it: policies in
 * sortPolicies order (src/policy-evaluator.ts:36-42), regex tests as HIT(rule, role) leaves (role 0 message, 1 conversation
 * entry, 2 + k tool param paramRole[k]), every other test an atom evaluated on the host by the reference's own condition code
 * (evalCondition = evaluateConditions over one condition, src/conditions/index.ts).  patternRule / toolRule: the rule of each
 * messageContains / conversationContains pattern and of each valid `matches` pattern in the scanner's rule set. */
type Ctx = Record<string, any>;
type Cond = Record<string, any>;
const OP = { CONST: 0, ATOM: 1, HIT: 2, AND: 3, OR: 4, NOT: 5 };
const ACTION: Record<string, number> = { allow: 0, audit: 1, "2fa": 2, deny: 3 };
const TIERS = ["untrusted", "restricted", "standard", "trusted", "elevated"];
export function compilePolicyProgram(policies: any[], patternRule: Map<string, number>, toolRule: Map<string, number>,
                                     evalCondition: (c: Cond, ctx: Ctx) => boolean) {
  const atomId = new Map<string, number>();
  const atoms: ((ctx: Ctx) => boolean)[] = [];
  const paramRole = new Map<string, number>();
  const atomIndex = (key: string, fn: (ctx: Ctx) => boolean) => {
    if (!atomId.has(key)) { atomId.set(key, atoms.length); atoms.push(fn); }
    return atomId.get(key)!;
  };
  const atom = (c: Cond) => [OP.ATOM | (atomIndex(JSON.stringify(c), (ctx) => evalCondition(c, ctx)) << 3)];
  const hit = (rule: number, role: number) => [(OP.HIT | (rule << 3) | (role << 24)) >>> 0];
  const fold = (parts: number[][], op: number, empty: number) =>
    parts.length ? parts.slice(1).reduce((acc, q) => [...acc, ...q, op], parts[0]) : [OP.CONST | (empty << 3)];
  const list = (v: any) => (Array.isArray(v) ? v : [v]);
  const cond = (c: Cond): number[] => {
    const parts: number[][] = [];
    if (c.type === "context") {
      for (const [key, role] of [["conversationContains", 1], ["messageContains", 0]] as const)
        if (c[key] != null) parts.push(fold(list(c[key]).map((p: string) => hit(patternRule.get(p)!, role)), OP.OR, 0));
      for (const key of ["hasMetadata", "channel", "sessionKey"]) if (c[key] != null) parts.push(atom({ type: "context", [key]: c[key] }));
      return fold(parts, OP.AND, 1);
    }
    if (c.type === "tool") {
      if (c.name != null) parts.push(atom({ type: "tool", name: c.name }));
      if (c.params && Object.keys(c.params).length) {
        for (const [key, m] of Object.entries<any>(c.params)) {
          if ("matches" in m && !("equals" in m) && !("contains" in m)) {
            if (!paramRole.has(key)) paramRole.set(key, 2 + paramRole.size);
            parts.push(toolRule.has(m.matches) ? hit(toolRule.get(m.matches)!, paramRole.get(key)!) : [OP.CONST]);
          } else parts.push(atom({ type: "tool", params: { [key]: m } }));
        }
      }
      return fold(parts, OP.AND, 1);
    }
    if (c.type === "agent") {
      for (const key of ["id", "trustTier"]) if (c[key] != null) parts.push(atom({ type: "agent", [key]: c[key] }));
      return fold(parts, OP.AND, 1);
    }
    if (c.type === "any") return fold((c.conditions ?? []).map(cond), OP.OR, 0);
    if (c.type === "not") return [...cond(c.condition), OP.NOT];
    return atom(c);                                           // time / risk / frequency
  };
  const spec = (p: any) => (p.scope?.agents?.length ? 10 : 0) + (p.scope?.channels?.length ? 5 : 0) + (p.scope?.hooks?.length ? 3 : 0);
  const order = [...policies].sort((a, b) => (b.priority ?? 0) - (a.priority ?? 0) || spec(b) - spec(a));
  const words: number[] = [order.length];
  const rules: [any, any][] = [];
  for (const p of order) {
    const sc = p.scope ?? {};
    words.push(sc.excludeAgents?.length || sc.channels?.length
      ? atomIndex("scope:" + JSON.stringify([sc.excludeAgents, sc.channels]), (ctx) =>
          !sc.excludeAgents?.includes(ctx.agentId) && !(sc.channels?.length && (!ctx.channel || !sc.channels.includes(ctx.channel))))
      : 0xffffffff, p.rules.length);
    for (const r of p.rules) {
      const tier = (ctx: Ctx) => TIERS.indexOf(ctx.trust?.session?.tier ?? "standard");
      const gates: number[][] = [];
      if (r.minTrust) gates.push([OP.ATOM | (atomIndex("minTrust:" + r.minTrust, (ctx) => tier(ctx) >= TIERS.indexOf(r.minTrust)) << 3)]);
      if (r.maxTrust) gates.push([OP.ATOM | (atomIndex("maxTrust:" + r.maxTrust, (ctx) => tier(ctx) <= TIERS.indexOf(r.maxTrust)) << 3)]);
      const ops = fold([...gates, ...(r.conditions ?? []).map(cond)], OP.AND, 1);
      words.push((ACTION[r.effect?.action] ?? 0) | (r.effect?.reason ? 4 : 0), ops.length, ...ops);
      rules.push([p, r]);
    }
  }
  return { program: Uint32Array.from(words), atoms, paramRole, rules };
}

/** Drop-in for PolicyEvaluator.evaluate (src/policy-evaluator.ts:18-146) on the hooks that evaluate one context per event
 * (before_tool_call, message_sending): the policies compiled once into a program on one rule set of their regex tests, then
 * per context its texts and atom row in one blocking call, one device round trip.  evalCondition: the reference's own
 * condition code for one condition (the atoms), as for compilePolicyProgram. */
export class GpuPolicyEvaluator {
  private readonly handle: unknown;
  private readonly compiled: ReturnType<typeof compilePolicyProgram>;

  constructor(policies: any[], evalCondition: (c: Cond, ctx: Ctx) => boolean) {
    const enabled = policies.filter((p) => p.enabled !== false);
    // one rule per messageContains / conversationContains pattern (an invalid one as an escaped literal, the includes()
    // fallback of context.ts:15-17), then one per valid tool `matches` pattern (an invalid one never matches, tool.ts:39-44)
    const patternRule = new Map<string, number>(), toolRule = new Map<string, number>(), toolPats = new Set<string>();
    const sources: { source: string }[] = [];
    const walk = (c: Cond): void => {
      if (c.type === "context") {
        for (const key of ["messageContains", "conversationContains"])
          for (const p of c[key] == null ? [] : Array.isArray(c[key]) ? c[key] : [c[key]])
            if (!patternRule.has(p)) {
              patternRule.set(p, sources.length);
              sources.push({ source: addon.ruleCheck(p) === -4 /* CG_ERR_SYNTAX */ ? p.replace(/[.*+?^${}()|[\]\\\/-]/g, "\\$&") : p });
            }
      } else if (c.type === "tool") {
        for (const m of Object.values<any>(c.params ?? {})) if ("matches" in m) toolPats.add(m.matches);
      } else if (c.type === "any") (c.conditions ?? []).forEach(walk);
      else if (c.type === "not") walk(c.condition);
    };
    for (const p of enabled) for (const r of p.rules ?? []) (r.conditions ?? []).forEach(walk);
    for (const p of [...toolPats].sort())
      if (addon.ruleCheck(p) === 0) { toolRule.set(p, sources.length); sources.push({ source: p }); }
    this.handle = addon.createRuleset(sources).handle;
    this.compiled = compilePolicyProgram(enabled, patternRule, toolRule, evalCondition);
    addon.setPolicyProgram(this.handle, this.compiled.program, this.compiled.atoms.length);
  }

  evaluate(ctx: Ctx): { action: string; reason: string; matches: { policyId: string; ruleId: string; effect: any; controls: string[] }[] } {
    const { atoms, paramRole, rules } = this.compiled;
    // the texts a leaf can read: a non-empty message (role 0), every conversation entry (1), string params a `matches` test names
    const texts: string[] = [], roleOf: number[] = [];
    if (ctx.messageContent) { texts.push(ctx.messageContent); roleOf.push(0); }
    for (const t of ctx.conversationContext ?? []) { texts.push(t); roleOf.push(1); }
    for (const [key, val] of Object.entries<any>(ctx.toolParams ?? {}))
      if (typeof val === "string" && paramRole.has(key)) { texts.push(val); roleOf.push(paramRole.get(key)!); }
    const row = new Uint32Array((atoms.length + 31) >>> 5);
    atoms.forEach((fn, a) => { if (fn(ctx)) row[a >>> 5] |= 1 << (a & 31); });
    const { bytes, offsets } = pack(texts);
    const { verdict, rules: hit } = addon.policyEvalOne(this.handle, bytes, offsets, Uint8Array.from(roleOf), row, atoms.length);
    // decode as plugin.PolicyEvaluator.decode_verdicts: outcome, deciding rule, the reference's reason strings
    const matches = Array.from(hit, (j) => {
      const [p, r] = rules[j];
      return { policyId: p.id, ruleId: r.id, effect: r.effect ?? { action: "allow" }, controls: p.controls ?? [] };
    });
    const outcome = verdict & 7, decide = verdict >>> 12;
    if (outcome >= 3) {
      const reason = decide !== 0xfffff ? rules[decide][1].effect.reason : outcome === 4 ? "Denied by governance policy" : "Requires 2FA approval";
      return { action: outcome === 4 ? "deny" : "2fa", reason, matches };
    }
    return { action: "allow", reason: ["No matching policies", "Allowed by governance policy", "Allowed with audit logging"][outcome], matches };
  }
}

/** sha256 (src/util.ts:77-79) for a batch of strings, hex digests. */
export function sha256Batch(texts: string[]): string[] {
  const parts = texts.map((t) => enc.encode(t));
  const offsets = new BigUint64Array(parts.length + 1);
  parts.forEach((p, i) => (offsets[i + 1] = offsets[i] + BigInt(p.length)));
  const bytes = new Uint8Array(Number(offsets[parts.length]) + 64);
  parts.forEach((p, i) => bytes.set(p, Number(offsets[i])));
  const d = addon.sha256Batch(bytes, offsets);
  return texts.map((_, i) => Buffer.from(d.subarray(32 * i, 32 * i + 32)).toString("hex"));
}

/** Proof-of-Guardrails: the day's audit JSONL (src/audit-trail.ts:151-179) as an append-only Merkle log.  flush() hands the
 * bytes it has just appended to the file to append(); root / frontier go next to the day file. */
export class AuditMerkleLog {
  private readonly log: unknown;
  constructor(restored?: { size: bigint; frontier: Uint8Array }) {
    this.log = restored ? addon.logRestore(restored.size, restored.frontier) : addon.logCreate(true);
  }
  append(flushedBytes: Uint8Array): bigint { return addon.logAppendJsonl(this.log, flushedBytes); }
  root(): string { return Buffer.from(addon.logRoot(this.log)).toString("hex"); }
  state(): { size: bigint; frontier: Uint8Array } { return { size: addon.logSize(this.log), frontier: addon.logFrontier(this.log) }; }
  inclusionProof(index: bigint): Uint8Array { return addon.logProof(this.log, index); }
  consistencyProof(firstSize: bigint): Uint8Array { return addon.logConsistency(this.log, firstSize); }
}

/** The same log keeping every complete subtree node (logCreateTree): an auditor holding yesterday's (size, root) gets receipts
 * for any records against that size, many per call, and checks a day's receipts in one call (RFC 6962 / RFC 9162). */
export class AuditMerkleTreeLog {
  private readonly log: unknown = addon.logCreateTree();
  append(flushedBytes: Uint8Array): bigint { return addon.logAppendJsonl(this.log, flushedBytes); }
  root(): string { return Buffer.from(addon.logRoot(this.log)).toString("hex"); }
  /** one audit path per index against the tree of the first treeSize records, leaf level first */
  inclusionProofs(indices: bigint[], treeSize: bigint): Uint8Array[] {
    const { paths, lens } = addon.logProofs(this.log, BigUint64Array.from(indices), treeSize);
    const stride = indices.length ? paths.length / 32 / indices.length : 0;
    return indices.map((_, i) => paths.subarray(32 * stride * i, 32 * (stride * i + lens[i])));
  }
  consistencyProof(firstSize: bigint, secondSize: bigint): Uint8Array { return addon.logConsistencyBetween(this.log, firstSize, secondSize); }
}

/** RFC 9162 2.1.3.2 for many receipts against one (treeSize, root): records as written by flush() (one JSON line each,
 * without its "\n"), their indices and paths -> per receipt whether it holds. */
export function verifyInclusionProofs(records: string[], indices: bigint[], treeSize: bigint, paths: Uint8Array[], root: Uint8Array): boolean[] {
  const parts = records.map((t) => enc.encode(t));
  const offsets = new BigUint64Array(parts.length + 1);
  parts.forEach((p, i) => (offsets[i + 1] = offsets[i] + BigInt(p.length)));
  const bytes = new Uint8Array(Number(offsets[parts.length]) + 64);
  parts.forEach((p, i) => bytes.set(p, Number(offsets[i])));
  const stride = Math.max(1, ...paths.map((p) => p.length / 32));
  const flat = new Uint8Array(paths.length * stride * 32);
  paths.forEach((p, i) => flat.set(p, 32 * stride * i));
  const lens = Uint32Array.from(paths.map((p) => p.length / 32));
  const ok = addon.verifyProofs(bytes, offsets, BigUint64Array.from(indices), treeSize, flat, lens, stride, root);
  return Array.from(ok, (v) => v !== 0);
}
