// expr.cu — FilterAndProjectOperator / PageProcessor on the GPU.
//
// Reference: PageProcessor.createWorkProcessor (M/operator/project/PageProcessor.java:105-142): evaluate
// the filter to SelectedPositions, then every projection over the selected positions
// (ProjectSelectedPositions.processBatch :302-336); FilterAndProjectOperator
// (M/operator/FilterAndProjectOperator.java:60-95) wraps it.  Output rows keep input order.
#include "expr.cuh"
#include "jit.cuh"

#include <algorithm>

namespace tg {

// strict UTF-8 -> UTF-16 code units (a Java String); false on malformed input
static bool utf8_to_utf16(const tgpu_bytes& b, std::u16string* out)
{
    out->clear();
    const uint8_t* p = b.data;
    int i = 0;
    while (i < b.length) {
        const int h = p[i];
        int n = h < 0x80 ? 0 : (h & 0xE0) == 0xC0 ? 1 : (h & 0xF0) == 0xE0 ? 2 : (h & 0xF8) == 0xF0 ? 3 : -1;
        if (n < 0 || i + n >= b.length) return false;
        uint32_t cp = n == 0 ? h : n == 1 ? (h & 0x1F) : n == 2 ? (h & 0x0F) : (h & 0x07);
        for (int k = 1; k <= n; k++) {
            if ((p[i + k] & 0xC0) != 0x80) return false;
            cp = (cp << 6) | (p[i + k] & 0x3F);
        }
        static const uint32_t min_cp[4] = {0, 0x80, 0x800, 0x10000};
        if (cp < min_cp[n] || cp > 0x10FFFF || (cp >= 0xD800 && cp <= 0xDFFF)) return false;
        if (cp >= 0x10000) {
            out->push_back((char16_t)(0xD800 + ((cp - 0x10000) >> 10)));
            out->push_back((char16_t)(0xDC00 + ((cp - 0x10000) & 0x3FF)));
        }
        else out->push_back((char16_t)cp);
        i += n + 1;
    }
    return true;
}

static void utf16_to_utf8(const std::u16string& s, std::string* out)
{
    out->clear();
    for (size_t i = 0; i < s.size(); i++) {
        uint32_t cp = s[i];
        if (cp >= 0xD800 && cp <= 0xDBFF && i + 1 < s.size()) cp = 0x10000 + ((cp - 0xD800) << 10) + (s[++i] - 0xDC00);
        if (cp < 0x80) *out += (char)cp;
        else if (cp < 0x800) { *out += (char)(0xC0 | (cp >> 6)); *out += (char)(0x80 | (cp & 0x3F)); }
        else if (cp < 0x10000) { *out += (char)(0xE0 | (cp >> 12)); *out += (char)(0x80 | ((cp >> 6) & 0x3F)); *out += (char)(0x80 | (cp & 0x3F)); }
        else {
            *out += (char)(0xF0 | (cp >> 18)); *out += (char)(0x80 | ((cp >> 12) & 0x3F));
            *out += (char)(0x80 | ((cp >> 6) & 0x3F)); *out += (char)(0x80 | (cp & 0x3F));
        }
    }
}

struct LikeItem {
    enum { LITERAL, ANY, ZERO_OR_MORE } kind;
    std::u16string literal;
    int count = 0;
};

// LikeMatcher.parse (M/likematcher/LikeMatcher.java:196-274); false where it throws (an invalid escape use)
static bool like_parse(const std::u16string& pat, int escape, std::vector<LikeItem>* out)
{
    std::u16string literal;
    int any = 0;
    bool unbounded = false, in_escape = false;
    auto flush_wild = [&] {
        if (any) { out->push_back(LikeItem{LikeItem::ANY, {}, any}); any = 0; }
        if (unbounded) { out->push_back(LikeItem{LikeItem::ZERO_OR_MORE, {}, 0}); unbounded = false; }
    };
    for (char16_t ch : pat) {
        if (in_escape) {
            if (ch != u'%' && ch != u'_' && (int)ch != escape) return false;
            literal += ch;
            in_escape = false;
        }
        else if (escape >= 0 && (int)ch == escape) {
            in_escape = true;
            flush_wild();
        }
        else if (ch == u'%' || ch == u'_') {
            if (!literal.empty()) { out->push_back(LikeItem{LikeItem::LITERAL, literal, 0}); literal.clear(); }
            if (ch == u'%') unbounded = true;
            else any++;
        }
        else {
            flush_wild();
            literal += ch;
        }
    }
    if (in_escape) return false;
    if (!literal.empty()) out->push_back(LikeItem{LikeItem::LITERAL, literal, 0});
    else flush_wild();
    return true;
}

// LikeMatcher.compile(pattern, escape, optimize = true) into the device form (device_lib.cuh DLike)
static int like_compile(tgpu_ctx* ctx, int idx, const tgpu_like_pattern& lp, DLike* L)
{
    memset(L, 0, sizeof(*L));
    if (lp.pattern.length < 0 || (lp.pattern.length > 0 && !lp.pattern.data) || lp.escape.length < 0 || (lp.escape.length > 0 && !lp.escape.data))
        return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "LIKE pattern %d: bad byte string", idx);
    std::u16string pat, esc;
    if (!utf8_to_utf16(lp.pattern, &pat)) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "LIKE pattern %d is not UTF-8", idx);
    if (!utf8_to_utf16(lp.escape, &esc)) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "LIKE escape %d is not UTF-8", idx);
    if (esc.size() > 1) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "LIKE pattern %d: the escape is not a single character", idx);
    std::vector<LikeItem> items;
    if (!like_parse(pat, esc.empty() ? -1 : (int)esc[0], &items))
        return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "LIKE pattern %d: escape character must be followed by '%%', '_' or the escape character itself", idx);
    std::vector<std::string> bytes(items.size());
    int64_t min_size = 0, max_size = 0;
    bool unbounded = false;
    for (size_t i = 0; i < items.size(); i++) {
        if (items[i].kind == LikeItem::LITERAL) {
            utf16_to_utf8(items[i].literal, &bytes[i]);
            min_size += (int64_t)bytes[i].size();
            max_size += (int64_t)bytes[i].size();
        }
        else if (items[i].kind == LikeItem::ANY) { min_size += items[i].count; max_size += 4LL * items[i].count; }
        else unbounded = true;
    }
    if (max_size > INT32_MAX) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "LIKE pattern %d is past the device limits", idx);
    L->min_size = (int32_t)min_size;
    L->max_size = unbounded ? -1 : (int32_t)max_size;
    int start = 0, end = (int)items.size() - 1;
    std::string stored;
    if (!items.empty() && items[0].kind == LikeItem::LITERAL) { stored += bytes[0]; L->prefix_len = (int32_t)bytes[0].size(); start++; }
    if (items.size() > 1 && items.back().kind == LikeItem::LITERAL) { stored += bytes.back(); L->suffix_len = (int32_t)bytes.back().size(); end--; }
    L->exact = 1;
    if (start <= end && items[end].kind == LikeItem::ZERO_OR_MORE) { L->exact = 0; end--; }
    L->kind = TGD_LIKE_NONE;
    if (start <= end) {
        bool has_any = false, any_after_zom = false, zom = false;
        for (int i = start; i <= end; i++) {
            if (items[i].kind == LikeItem::ANY) { any_after_zom = zom; has_any = true; break; }
            if (items[i].kind == LikeItem::ZERO_OR_MORE) zom = true;
        }
        L->kind = !has_any ? TGD_LIKE_FJS : !any_after_zom ? TGD_LIKE_DFA : TGD_LIKE_NFA;
        int pos = 0;
        auto state = [&](int kind_bit, int val) -> bool {
            if (pos >= 63) return false;
            if (kind_bit) L->any_mask |= 1ULL << pos;
            else {
                if (L->num_lits >= TGD_LIKE_LITS) return false;
                L->lit_pos[L->num_lits] = pos;
                L->lit_val[L->num_lits++] = val;
            }
            pos++;
            return true;
        };
        for (int i = start; i <= end; i++) {
            const LikeItem& it = items[i];
            bool ok = true;
            if (L->kind == TGD_LIKE_FJS) {
                if (it.kind != LikeItem::LITERAL) continue;
                if (L->num_terms >= TGD_LIKE_TERMS) ok = false;
                else {
                    L->term_off[L->num_terms] = (int32_t)stored.size();
                    L->term_len[L->num_terms++] = (int32_t)bytes[i].size();
                    stored += bytes[i];
                }
            }
            else if (it.kind == LikeItem::ZERO_OR_MORE) L->loop_mask |= 1ULL << pos;
            else if (it.kind == LikeItem::ANY) for (int k = 0; k < it.count && ok; k++) ok = state(1, 0);
            else if (L->kind == TGD_LIKE_DFA) for (unsigned char c : bytes[i]) { if (ok) ok = state(0, c); }
            else for (char16_t c : it.literal) { if (ok) ok = state(0, (int)c); }
            if (!ok) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "LIKE pattern %d needs more matcher states than the device form holds", idx);
        }
        L->accept = pos;
    }
    if (stored.size() > TGD_LIKE_BYTES) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "LIKE pattern %d holds more than %d literal bytes", idx, TGD_LIKE_BYTES);
    memcpy(L->bytes, stored.data(), stored.size());
    return TGPU_OK;
}

static bool varchar_op(int op)
{
    switch (op) {
        case TGPU_EX_EQ: case TGPU_EX_NE: case TGPU_EX_LT: case TGPU_EX_LE: case TGPU_EX_GT: case TGPU_EX_GE: case TGPU_EX_BETWEEN:
        case TGPU_EX_IN: case TGPU_EX_IS_NULL: case TGPU_EX_IS_NOT_NULL: case TGPU_EX_LIKE:
        case TGPU_EX_LENGTH: case TGPU_EX_SUBSTR: case TGPU_EX_LTRIM: case TGPU_EX_RTRIM: case TGPU_EX_TRIM: case TGPU_EX_CONCAT:
            return true;
        default: return false;
    }
}

static bool string_function(int op) { return op >= TGPU_EX_LENGTH && op <= TGPU_EX_CONCAT; }

// the vtype of what instruction `s` writes to its temp
static int result_vtype(const tgpu_expr_insn& s)
{
    switch (s.op) {
        case TGPU_EX_EQ: case TGPU_EX_NE: case TGPU_EX_LT: case TGPU_EX_LE: case TGPU_EX_GT: case TGPU_EX_GE: case TGPU_EX_AND: case TGPU_EX_OR:
        case TGPU_EX_NOT: case TGPU_EX_IS_NULL: case TGPU_EX_IS_NOT_NULL: case TGPU_EX_BETWEEN: case TGPU_EX_IN: case TGPU_EX_LIKE:
            return TGPU_V_BOOLEAN;
        case TGPU_EX_CAST_BIGINT_TO_DOUBLE: case TGPU_EX_CAST_DECIMAL_TO_DOUBLE: return TGPU_V_DOUBLE;
        case TGPU_EX_CAST_DOUBLE_TO_BIGINT: case TGPU_EX_CAST_DECIMAL_TO_BIGINT: case TGPU_EX_LENGTH: return TGPU_V_BIGINT;
        case TGPU_EX_CAST_TO_DECIMAL: return TGPU_V_DECIMAL;
        default: return s.vtype;
    }
}

// What each temp holds while the instructions are compiled in order
struct TempState {
    int vt[TGPU_MAX_TEMPS];         // vtype of the value, -1 never written
    int kind[TGPU_MAX_TEMPS];       // VARCHAR temps: 1 a view, 2 a CONCAT result
    int32_t src[TGPU_MAX_TEMPS];    // a view's source
    int cat[TGPU_MAX_TEMPS];        // a CONCAT result's instruction
    TempState() { for (int t = 0; t < TGPU_MAX_TEMPS; t++) { vt[t] = -1; kind[t] = 0; src[t] = TGD_SRC_NONE; cat[t] = -1; } }
};

// one instruction with VARCHAR operands: operands are UTF8 channels (given a string slot), pool constants, NULL, or temps holding a
// VARCHAR (a view, or a CONCAT result that only CONCAT reads).  SUBSTR's start and length are BIGINT operands.
static int compile_varchar_insn(tgpu_ctx* ctx, const tgpu_expr_program* p, int i, DProgram* out, int32_t* max_channel, TempState* ts)
{
    const tgpu_expr_insn& s = p->insns[i];
    DInsn& d = out->insns[i];
    if (s.vtype != TGPU_V_VARCHAR) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: LIKE needs VARCHAR operands", i);
    if (!varchar_op(s.op)) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: op %d does not take VARCHAR operands", i, s.op);
    if (s.dst < 0 || s.dst >= TGPU_MAX_TEMPS) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: dst temp out of range", i);
    const bool unary = s.op == TGPU_EX_IS_NULL || s.op == TGPU_EX_IS_NOT_NULL || s.op == TGPU_EX_IN || s.op == TGPU_EX_LIKE || s.op == TGPU_EX_LENGTH ||
                       s.op == TGPU_EX_LTRIM || s.op == TGPU_EX_RTRIM || s.op == TGPU_EX_TRIM;
    const tgpu_operand* ops[3] = {&s.a, &s.b, &s.c};
    DOperand* dops[3] = {&d.a, &d.b, &d.c};
    const int used = unary ? 1 : (s.op == TGPU_EX_BETWEEN || (s.op == TGPU_EX_SUBSTR && s.c.kind != TGPU_OPND_NONE)) ? 3 : 2;
    for (int k = 0; k < 3; k++) {
        const tgpu_operand& o = *ops[k];
        DOperand& x = *dops[k];
        x.kind = k < used ? o.kind : TGPU_OPND_NONE;
        x.index = o.index;
        x.imm = o.imm.i64;
        if (k >= used) continue;
        if (s.op == TGPU_EX_SUBSTR && k > 0) {
            // the BIGINT start and length
            if (o.kind == TGPU_OPND_TEMP) {
                if (o.index < 0 || o.index >= TGPU_MAX_TEMPS) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "operand temp %d out of range", o.index);
                if (ts->vt[o.index] != TGPU_V_BIGINT) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: substr's start and length are BIGINT", i);
            }
            else if (o.kind == TGPU_OPND_COLUMN) {
                if (o.index < 0 || o.index >= TGPU_MAX_CHANNELS) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "operand channel %d out of range", o.index);
                if (o.index > *max_channel) *max_channel = o.index;
            }
            else if (o.kind != TGPU_OPND_CONST && o.kind != TGPU_OPND_NULL) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: bad BIGINT operand kind %d", i, o.kind);
            continue;
        }
        if (o.kind == TGPU_OPND_TEMP) {
            if (o.index < 0 || o.index >= TGPU_MAX_TEMPS || ts->vt[o.index] != TGPU_V_VARCHAR)
                return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: a VARCHAR temp operand must be written by an earlier VARCHAR instruction", i);
            if (ts->kind[o.index] == 2 && s.op != TGPU_EX_CONCAT)
                return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "insn %d: a concatenation is read only by another concatenation or a projection", i);
            x.imm = ts->src[o.index];
        }
        else if (o.kind == TGPU_OPND_CONST) {
            if (o.imm.i64 < 0 || o.imm.i64 >= p->num_strings) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: pool string index out of range", i);
        }
        else if (o.kind == TGPU_OPND_COLUMN) {
            if (o.index < 0 || o.index >= TGPU_MAX_CHANNELS) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "operand channel %d out of range", o.index);
            if (o.index > *max_channel) *max_channel = o.index;
            if (out->str_slot[o.index] < 0) {
                if (out->num_str_channels >= TGD_MAX_STR_CHANNELS)
                    return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "string operations read more than %d VARCHAR channels", TGD_MAX_STR_CHANNELS);
                out->str_slot[o.index] = (int8_t)out->num_str_channels;
                out->str_channel[out->num_str_channels++] = o.index;
            }
        }
        else if (o.kind != TGPU_OPND_NULL) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: bad VARCHAR operand kind %d", i, o.kind);
    }
    if (s.op == TGPU_EX_IN) {
        if (s.b.imm.i64 < 0 || s.b.imm.i64 >= p->num_in_lists) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: IN list index out of range", i);
        const tgpu_in_list& l = p->in_lists[s.b.imm.i64];
        for (int k = 0; k < l.count; k++)
            if (l.values[k] < 0 || l.values[k] >= p->num_strings) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: pool string index out of range", i);
    }
    if (s.op == TGPU_EX_LIKE && (s.b.imm.i64 < 0 || s.b.imm.i64 >= p->num_like_patterns))
        return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: LIKE pattern index out of range", i);
    if (s.op == TGPU_EX_IN || s.op == TGPU_EX_LIKE) { d.b.kind = TGPU_OPND_CONST; d.b.imm = s.b.imm.i64; }
    d.op = s.op;
    d.vtype = s.vtype;
    d.dst = s.dst;
    if (string_function(s.op)) out->has_strfn = 1;
    // the source of a VARCHAR operand's bytes
    auto src_of = [&](const DOperand& o) -> int32_t {
        if (o.kind == TGPU_OPND_COLUMN) return o.index;
        if (o.kind == TGPU_OPND_CONST) return (int32_t)(-(o.imm + 1));
        if (o.kind == TGPU_OPND_TEMP) return (int32_t)o.imm;
        return TGD_SRC_NONE;
    };
    int kind = 0, cat = -1;
    int32_t src = TGD_SRC_NONE;
    if (s.op == TGPU_EX_SUBSTR || s.op == TGPU_EX_LTRIM || s.op == TGPU_EX_RTRIM || s.op == TGPU_EX_TRIM) {
        kind = 1;
        src = src_of(d.a);
    }
    else if (s.op == TGPU_EX_CONCAT) {
        DCat& c = out->cat[i];
        memset(&c, 0, sizeof(c));
        c.a_slot = c.b_slot = -1;
        const DOperand* cops[2] = {&d.a, &d.b};
        int8_t* capture[2] = {&c.a_slot, &c.b_slot};
        for (int k = 0; k < 2; k++) {
            const DOperand& o = *cops[k];
            if (o.kind == TGPU_OPND_TEMP && ts->kind[o.index] == 2) {
                DCat& inner = out->cat[ts->cat[o.index]];
                inner.inner = 1;
                for (int q = 0; q < inner.n; q++) {
                    if (c.n >= TGD_MAX_PIECES) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "insn %d: a concatenation of more than %d pieces", i, TGD_MAX_PIECES);
                    c.slot[c.n] = inner.slot[q];
                    c.src[c.n++] = inner.src[q];
                }
                continue;
            }
            if (c.n >= TGD_MAX_PIECES) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "insn %d: a concatenation of more than %d pieces", i, TGD_MAX_PIECES);
            if (out->num_piece_slots >= TGD_MAX_PIECE_SLOTS)
                return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "concatenations capture more than %d pieces", TGD_MAX_PIECE_SLOTS);
            *capture[k] = (int8_t)out->num_piece_slots;
            c.slot[c.n] = (int8_t)out->num_piece_slots++;
            c.src[c.n++] = src_of(o);
        }
        kind = 2;
        cat = i;
    }
    ts->vt[s.dst] = result_vtype(s);
    ts->kind[s.dst] = kind;
    ts->src[s.dst] = src;
    ts->cat[s.dst] = cat;
    return TGPU_OK;
}

// ---- DECIMAL ------------------------------------------------------------------------------------------------------------------------
struct DecType {
    int p = 0, s = 0;     // p == 0: not a DECIMAL
    bool operator==(const DecType& o) const { return p == o.p && s == o.s; }
    bool lng() const { return p > 18; }
};

static bool dec_insn(const tgpu_expr_insn& s)
{
    return s.vtype == TGPU_V_DECIMAL || s.op == TGPU_EX_CAST_TO_DECIMAL || s.op == TGPU_EX_CAST_DECIMAL_TO_BIGINT || s.op == TGPU_EX_CAST_DECIMAL_TO_DOUBLE;
}

static long long pow10_i64(int k)
{
    long long r = 1;
    for (int i = 0; i < k; i++) r *= 10;
    return r;
}

// the DECIMAL instructions of `p`: every type checked against the rules of the signatures, and the reference's method of each
// (DecimalOperators.java's specialisers: calculateShortRescaleParameters, calculateLongRescaleParameters,
// calculateMultiplicativeResultRescale, divideRescaleFactor; DecimalCasts / DecimalToDecimalCasts) fixed in out->dec
static int compile_decimals(tgpu_ctx* ctx, const tgpu_expr_program* p, DProgram* out)
{
    bool any = false;
    for (int i = 0; i < p->num_insns; i++) any = any || dec_insn(p->insns[i]);
    if (!any) return TGPU_OK;
    if (!p->decimal_signatures) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "a program with DECIMAL instructions needs decimal_signatures");
    if (p->num_decimal_constants < 0 || (p->num_decimal_constants > 0 && !p->decimal_constants))
        return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "bad decimal constants");
    out->has_dec = 1;
    DecType temp_t[TGPU_MAX_TEMPS], col_t[TGPU_MAX_CHANNELS];
    bool temp_written[TGPU_MAX_TEMPS] = {false};
    int8_t col_seen[TGPU_MAX_CHANNELS] = {0};     // 1 read as a DECIMAL, 2 as something else
    auto valid = [](const tgpu_decimal_type& t) { return t.precision >= 1 && t.precision <= 38 && t.scale >= 0 && t.scale <= t.precision; };
    // does a value fit DECIMAL(t)?  (hi, lo) two's complement
    auto fits = [](const DecType& t, long long hi, long long lo) {
        const U128 v{(unsigned long long)hi, (unsigned long long)lo};
        return !u128_exceeds_precision(v, t.p);
    };
    for (int i = 0; i < p->num_insns; i++) {
        const tgpu_expr_insn& s = p->insns[i];
        DInsn& d = out->insns[i];
        const tgpu_operand* ops[3] = {&s.a, &s.b, &s.c};
        DOperand* dops[3] = {&d.a, &d.b, &d.c};
        const bool unary = s.op == TGPU_EX_MOV || s.op == TGPU_EX_NEG || s.op == TGPU_EX_IS_NULL || s.op == TGPU_EX_IS_NOT_NULL || s.op == TGPU_EX_IN ||
                           s.op == TGPU_EX_CAST_TO_DECIMAL || s.op == TGPU_EX_CAST_DECIMAL_TO_BIGINT || s.op == TGPU_EX_CAST_DECIMAL_TO_DOUBLE ||
                           s.op == TGPU_EX_NOT;
        const int used = unary ? 1 : (s.op == TGPU_EX_BETWEEN || s.op == TGPU_EX_IF) ? 3 : 2;
        if (!dec_insn(s)) {
            // a numeric instruction never reads a DECIMAL temp or a channel read as DECIMAL
            for (int k = 0; k < used && k < 3; k++) {
                if (s.op == TGPU_EX_IN && k > 0) break;
                if (ops[k]->kind == TGPU_OPND_TEMP && temp_t[ops[k]->index].p)
                    return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d reads DECIMAL temp %d as another type", i, ops[k]->index);
                if (ops[k]->kind == TGPU_OPND_COLUMN && s.vtype != TGPU_V_VARCHAR && s.op != TGPU_EX_LIKE) {
                    if (col_seen[ops[k]->index] == 1) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d reads DECIMAL channel %d as another type", i, ops[k]->index);
                    col_seen[ops[k]->index] = 2;
                }
            }
            temp_t[s.dst] = DecType{};
            temp_written[s.dst] = true;
            continue;
        }
        const tgpu_decimal_signature& sig = p->decimal_signatures[i];
        DDec& x = out->dec[i];
        memset(&x, 0, sizeof(x));
        x.is_dec = 1;
        // which operands and result are DECIMAL
        bool opnd_dec = s.vtype == TGPU_V_DECIMAL;
        bool res_dec = false;
        switch (s.op) {
            case TGPU_EX_MOV: case TGPU_EX_ADD: case TGPU_EX_SUB: case TGPU_EX_MUL: case TGPU_EX_DIV: case TGPU_EX_NEG: res_dec = true; break;
            case TGPU_EX_EQ: case TGPU_EX_NE: case TGPU_EX_LT: case TGPU_EX_LE: case TGPU_EX_GT: case TGPU_EX_GE: case TGPU_EX_BETWEEN:
            case TGPU_EX_IN: case TGPU_EX_IS_NULL: case TGPU_EX_IS_NOT_NULL: break;
            case TGPU_EX_CAST_TO_DECIMAL:
                if (s.vtype == TGPU_V_DOUBLE) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "insn %d: CAST(DOUBLE AS DECIMAL) is not evaluated on the GPU", i);
                if (s.vtype != TGPU_V_BIGINT && s.vtype != TGPU_V_DECIMAL) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: CAST to DECIMAL reads BIGINT or DECIMAL", i);
                res_dec = true;
                break;
            case TGPU_EX_CAST_DECIMAL_TO_BIGINT: case TGPU_EX_CAST_DECIMAL_TO_DOUBLE:
                if (s.vtype != TGPU_V_DECIMAL) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: this cast reads a DECIMAL operand", i);
                break;
            case TGPU_EX_MOD: return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "insn %d: DECIMAL %% is not evaluated on the GPU", i);
            case TGPU_EX_IF: case TGPU_EX_COALESCE: res_dec = true; break;
            default: return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: op %d does not take DECIMAL operands", i, s.op);
        }
        // operand k is DECIMAL (IF's condition is a BOOLEAN: it keeps ot[0] = not a DECIMAL, so la = 0 and it is read as a plain word)
        auto dec_opnd = [&](int k) { return opnd_dec && !(s.op == TGPU_EX_IF && k == 0); };
        DecType ot[3], rt;
        const tgpu_decimal_type* st[3] = {&sig.a, &sig.b, &sig.c};
        const int nopnd = s.op == TGPU_EX_IN ? 1 : used;
        for (int k = 0; k < nopnd; k++) {
            if (!dec_opnd(k)) continue;
            if (!valid(*st[k])) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: bad DECIMAL type of operand %d", i, k);
            ot[k] = DecType{st[k]->precision, st[k]->scale};
        }
        if (res_dec) {
            if (!valid(sig.result)) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: bad DECIMAL result type", i);
            rt = DecType{sig.result.precision, sig.result.scale};
        }
        // operands: temps carry their writer's type, a channel one type throughout, constants fit their type
        for (int k = 0; k < nopnd; k++) {
            const tgpu_operand& o = *ops[k];
            if (o.kind == TGPU_OPND_TEMP) {
                if (!temp_written[o.index] || !(temp_t[o.index] == ot[k]))
                    return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: temp %d does not hold the operand's type", i, o.index);
            }
            else if (o.kind == TGPU_OPND_COLUMN) {
                if (!dec_opnd(k)) {
                    if (col_seen[o.index] == 1) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d reads DECIMAL channel %d as another type", i, o.index);
                    col_seen[o.index] = 2;
                }
                else {
                    if (col_seen[o.index] == 2 || (col_seen[o.index] == 1 && !(col_t[o.index] == ot[k])))
                        return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d reads channel %d with another type", i, o.index);
                    col_seen[o.index] = 1;
                    col_t[o.index] = ot[k];
                }
            }
            else if (o.kind == TGPU_OPND_CONST && dec_opnd(k)) {
                long long hi = o.imm.i64 >> 63, lo = o.imm.i64;
                if (ot[k].lng()) {
                    if (o.imm.i64 < 0 || o.imm.i64 >= p->num_decimal_constants)
                        return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: decimal constant index out of range", i);
                    hi = p->decimal_constants[2 * o.imm.i64];
                    lo = p->decimal_constants[2 * o.imm.i64 + 1];
                    x.hi[k] = hi;
                    dops[k]->imm = lo;
                }
                if (!fits(ot[k], hi, lo)) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: constant does not fit DECIMAL(%d, %d)", i, ot[k].p, ot[k].s);
            }
        }
        if (s.op == TGPU_EX_IN) {
            const tgpu_in_list& l = p->in_lists[s.b.imm.i64];
            const int off = out->in_offset[s.b.imm.i64];
            for (int k = 0; k < l.count; k++) {
                long long hi = l.values[k] >> 63, lo = l.values[k];
                if (ot[0].lng()) {
                    if (l.values[k] < 0 || l.values[k] >= p->num_decimal_constants)
                        return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: decimal constant index out of range", i);
                    hi = p->decimal_constants[2 * l.values[k]];
                    lo = p->decimal_constants[2 * l.values[k] + 1];
                }
                if (!fits(ot[0], hi, lo)) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: IN value does not fit DECIMAL(%d, %d)", i, ot[0].p, ot[0].s);
                out->in_values[off + k] = lo;
                out->in_hi[off + k] = hi;
            }
        }
        const bool cmp = s.op == TGPU_EX_EQ || s.op == TGPU_EX_NE || s.op == TGPU_EX_LT || s.op == TGPU_EX_LE || s.op == TGPU_EX_GT || s.op == TGPU_EX_GE ||
                         s.op == TGPU_EX_BETWEEN;
        if (cmp && !(ot[0] == ot[1] && (s.op != TGPU_EX_BETWEEN || ot[0] == ot[2])))
            return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: compared DECIMAL operands have different types", i);
        if ((s.op == TGPU_EX_MOV || s.op == TGPU_EX_NEG) && !(rt == ot[0]))
            return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: the result has another type than the operand", i);
        if ((s.op == TGPU_EX_IF && !(ot[1] == rt && ot[2] == rt)) || (s.op == TGPU_EX_COALESCE && !(ot[0] == rt && ot[1] == rt)))
            return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: the operands of IF / COALESCE and its result are not one DECIMAL type", i);
        x.la = ot[0].lng();
        x.lb = ot[1].lng();
        x.lc = ot[2].lng();
        x.lr = rt.lng();
        const bool any_long = x.la || x.lb;
        switch (s.op) {
            case TGPU_EX_ADD: case TGPU_EX_SUB: {
                const int ar = std::max(0, ot[1].s - ot[0].s), br = std::max(0, ot[0].s - ot[1].s);
                if (!any_long && !x.lr) { x.m0 = pow10_i64(ar); x.m1 = pow10_i64(br); }
                else {
                    if (!x.lr) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: a long operand needs a long result", i);
                    x.k0 = ar == 0 ? br : ar;
                    x.k1 = ar == 0 ? 0 : 1;
                    x.k2 = rt.s - std::max(ot[0].s, ot[1].s);
                }
                break;
            }
            case TGPU_EX_MUL:
                if (any_long && !x.lr) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: a long operand needs a long result", i);
                x.k2 = rt.s - (ot[0].s + ot[1].s);
                break;
            case TGPU_EX_DIV:
                x.k0 = rt.s - ot[0].s + ot[1].s;
                if (x.la && x.lb && !x.lr) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: DECIMAL long / long -> short has no method", i);
                if (!any_long && !x.lr) {
                    if (x.k0 < 0 || x.k0 > 18) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "insn %d: short DECIMAL division rescales by 10^%d", i, x.k0);
                    x.m0 = pow10_i64(x.k0);
                }
                break;
            case TGPU_EX_CAST_TO_DECIMAL:
                x.k0 = rt.p;
                if (s.vtype == TGPU_V_BIGINT) {
                    x.k1 = rt.s;
                    if (!x.lr) x.m0 = pow10_i64(rt.s);
                }
                else {
                    x.k1 = rt.s - ot[0].s;
                    x.k2 = rt == ot[0] ? 1 : 0;
                    if (!x.la && !x.lr) { x.m0 = pow10_i64(std::abs(x.k1)); x.m1 = x.m0 / 2; }
                }
                break;
            case TGPU_EX_CAST_DECIMAL_TO_BIGINT: case TGPU_EX_CAST_DECIMAL_TO_DOUBLE:
                x.k1 = ot[0].s;
                if (!x.la) x.m0 = pow10_i64(ot[0].s);
                break;
            default: break;
        }
        temp_t[s.dst] = res_dec ? rt : DecType{};
        temp_written[s.dst] = true;
        if (res_dec && rt.lng()) out->long_temps |= 1u << s.dst;
    }
    for (int t = 0; t < TGPU_MAX_TEMPS; t++) out->temp_dec[t] = temp_t[t].p == 0 ? 0 : temp_t[t].lng() ? 2 : 1;
    return TGPU_OK;
}

// IF / COALESCE (vtype not VARCHAR): IF's condition is BOOLEAN; the selected operands are present and, when temps, hold vtype (a channel's
// type is known only at add_input, a constant has no type of its own).  Runs before the instruction's own result is recorded in `ts`.
static int check_conditional(tgpu_ctx* ctx, const tgpu_expr_insn& s, int i, const TempState& ts)
{
    const bool is_if = s.op == TGPU_EX_IF;
    auto temp_vt = [&](const tgpu_operand& o) { return o.index >= 0 && o.index < TGPU_MAX_TEMPS ? ts.vt[o.index] : -1; };
    if (is_if && (s.a.kind == TGPU_OPND_NONE || (s.a.kind == TGPU_OPND_TEMP && temp_vt(s.a) != TGPU_V_BOOLEAN)))
        return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: the condition of IF is BOOLEAN", i);
    const tgpu_operand* sel[2] = {is_if ? &s.b : &s.a, is_if ? &s.c : &s.b};
    for (const tgpu_operand* o : sel) {
        if (o->kind == TGPU_OPND_NONE) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: IF / COALESCE is missing an operand", i);
        if (o->kind == TGPU_OPND_TEMP && temp_vt(*o) != s.vtype)
            return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: temp %d does not hold the vtype of IF / COALESCE", i, o->index);
    }
    return TGPU_OK;
}

bool expr_uses_strings(const DProgram& prog)
{
    for (int i = 0; i < prog.num_insns; i++)
        if (prog.insns[i].vtype == TGPU_V_VARCHAR || prog.insns[i].op == TGPU_EX_LIKE) return true;
    return false;
}

int expr_compile(tgpu_ctx* ctx, const tgpu_expr_program* p, DProgram* out, int32_t* max_channel)
{
    memset(out, 0, sizeof(*out));
    *max_channel = -1;
    if (!p) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "expression program is null");
    if (p->num_insns < 0 || p->num_insns > TGPU_MAX_INSNS) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "expression program has %d instructions (max %d)", p->num_insns, TGPU_MAX_INSNS);
    if (p->num_filter_insns < 0 || p->num_filter_insns > p->num_insns) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "num_filter_insns out of range");
    if (p->filter_temp >= TGPU_MAX_TEMPS) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "filter_temp out of range");
    if (p->num_in_lists > 8) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "more than 8 IN lists");
    out->num_insns = p->num_insns;
    out->num_filter_insns = p->filter_temp >= 0 ? p->num_filter_insns : 0;
    out->filter_temp = p->filter_temp;
    out->num_in_lists = p->num_in_lists;
    int off = 0;
    for (int i = 0; i < p->num_in_lists; i++) {
        if (off + p->in_lists[i].count > 128) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "IN lists hold more than 128 constants");
        out->in_offset[i] = off;
        out->in_count[i] = p->in_lists[i].count;
        for (int k = 0; k < p->in_lists[i].count; k++) out->in_values[off + k] = p->in_lists[i].values[k];
        off += p->in_lists[i].count;
    }
    memset(out->str_slot, -1, sizeof(out->str_slot));
    if (p->num_strings < 0 || (p->num_strings > 0 && !p->strings)) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "bad string pool");
    if (p->num_strings > TGPU_MAX_STRINGS) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "more than %d pool strings", TGPU_MAX_STRINGS);
    int64_t pool_bytes = 0;
    for (int k = 0; k < p->num_strings; k++) {
        const tgpu_bytes& b = p->strings[k];
        if (b.length < 0 || (b.length > 0 && !b.data)) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "pool string %d: bad byte string", k);
        if (pool_bytes + b.length > TGPU_MAX_STRING_BYTES) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "pool strings hold more than %d bytes", TGPU_MAX_STRING_BYTES);
        out->str_off[k] = (int32_t)pool_bytes;
        out->str_len[k] = b.length;
        if (b.length) memcpy(out->str_bytes + pool_bytes, b.data, (size_t)b.length);
        pool_bytes += b.length;
    }
    out->num_strings = p->num_strings;
    if (p->num_like_patterns < 0 || (p->num_like_patterns > 0 && !p->like_patterns)) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "bad LIKE patterns");
    if (p->num_like_patterns > TGPU_MAX_LIKE_PATTERNS) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "more than %d LIKE patterns", TGPU_MAX_LIKE_PATTERNS);
    for (int k = 0; k < p->num_like_patterns; k++) TG_TRY(like_compile(ctx, k, p->like_patterns[k], &out->likes[k]));
    out->num_likes = p->num_like_patterns;
    auto conv = [&](const tgpu_operand& o, DOperand* d) -> int {
        d->kind = o.kind;
        d->index = o.index;
        d->imm = o.imm.i64;
        if (o.kind == TGPU_OPND_COLUMN) {
            if (o.index < 0 || o.index >= TGPU_MAX_CHANNELS) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "operand channel %d out of range", o.index);
            if (o.index > *max_channel) *max_channel = o.index;
        }
        else if (o.kind == TGPU_OPND_TEMP) {
            if (o.index < 0 || o.index >= TGPU_MAX_TEMPS) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "operand temp %d out of range", o.index);
        }
        else if (o.kind < 0 || o.kind > TGPU_OPND_NULL) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "bad operand kind %d", o.kind);
        return TGPU_OK;
    };
    TempState ts;
    for (int i = 0; i < p->num_insns; i++) {
        const tgpu_expr_insn& s = p->insns[i];
        DInsn& d = out->insns[i];
        if (s.dst < 0 || s.dst >= TGPU_MAX_TEMPS) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: dst temp out of range", i);
        if (s.vtype < 0 || s.vtype > TGPU_V_DECIMAL) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: bad vtype", i);
        const bool cond = s.op == TGPU_EX_IF || s.op == TGPU_EX_COALESCE;
        // a VARCHAR temp is a view of one static source: a per-row choice between two sources does not fit it
        if (cond && s.vtype == TGPU_V_VARCHAR) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "insn %d: IF / COALESCE with a VARCHAR result is not evaluated on the GPU", i);
        if (cond) TG_TRY(check_conditional(ctx, s, i, ts));
        if (s.vtype == TGPU_V_VARCHAR || s.op == TGPU_EX_LIKE) {
            TG_TRY(compile_varchar_insn(ctx, p, i, out, max_channel, &ts));
            continue;
        }
        if (string_function(s.op)) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: a string function needs VARCHAR operands", i);
        for (const tgpu_operand* o : {&s.a, &s.b, &s.c})
            if (o->kind == TGPU_OPND_TEMP && o->index >= 0 && o->index < TGPU_MAX_TEMPS && ts.vt[o->index] == TGPU_V_VARCHAR && !(s.op == TGPU_EX_IN && o != &s.a))
                return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d reads VARCHAR temp %d as another type", i, o->index);
        ts.vt[s.dst] = result_vtype(s);
        ts.kind[s.dst] = 0;
        switch (s.op) {
            case TGPU_EX_MOV: case TGPU_EX_ADD: case TGPU_EX_SUB: case TGPU_EX_MUL: case TGPU_EX_DIV: case TGPU_EX_MOD: case TGPU_EX_NEG:
            case TGPU_EX_EQ: case TGPU_EX_NE: case TGPU_EX_LT: case TGPU_EX_LE: case TGPU_EX_GT: case TGPU_EX_GE:
            case TGPU_EX_AND: case TGPU_EX_OR: case TGPU_EX_NOT: case TGPU_EX_IS_NULL: case TGPU_EX_IS_NOT_NULL: case TGPU_EX_BETWEEN:
            case TGPU_EX_CAST_BIGINT_TO_DOUBLE: case TGPU_EX_CAST_DOUBLE_TO_BIGINT:
            case TGPU_EX_CAST_TO_DECIMAL: case TGPU_EX_CAST_DECIMAL_TO_BIGINT: case TGPU_EX_CAST_DECIMAL_TO_DOUBLE:
            case TGPU_EX_IF: case TGPU_EX_COALESCE:
                break;
            case TGPU_EX_IN:
                if (s.b.imm.i64 < 0 || s.b.imm.i64 >= p->num_in_lists) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: IN list index out of range", i);
                break;
            default:
                return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "insn %d: unsupported op %d", i, s.op);
        }
        d.op = s.op;
        d.vtype = s.vtype;
        d.dst = s.dst;
        TG_TRY(conv(s.a, &d.a));
        TG_TRY(conv(s.b, &d.b));
        TG_TRY(conv(s.c, &d.c));
        if (s.op == TGPU_EX_IN) d.b.kind = TGPU_OPND_CONST;
    }
    // VARCHAR projections: the view or the pieces the output is assembled from
    for (int k = 0; k < p->num_projections && p->projections; k++) {
        const tgpu_projection& pr = p->projections[k];
        if (pr.kind != 1 || pr.index < 0 || pr.index >= TGPU_MAX_TEMPS) continue;
        const int t = pr.index;
        if ((pr.vtype == TGPU_V_VARCHAR) != (ts.vt[t] == TGPU_V_VARCHAR && p->num_insns > 0))
            return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "projection %d: the projection's type and what temp %d holds differ", k, t);
        if (pr.vtype != TGPU_V_VARCHAR) continue;
        if (out->num_str_outs >= TGD_MAX_STR_OUTS) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "more than %d VARCHAR projections", TGD_MAX_STR_OUTS);
        DStrOut& so = out->str_out[out->num_str_outs++];
        memset(&so, 0, sizeof(so));
        so.temp = t;
        if (ts.kind[t] == 2) {
            const DCat& c = out->cat[ts.cat[t]];
            if (c.inner) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "projection %d: temp %d is also read by a later concatenation", k, t);
            so.n = c.n;
            for (int q = 0; q < c.n; q++) { so.slot[q] = c.slot[q]; so.src[q] = c.src[q]; }
        }
        else {
            so.n = 1;
            so.slot[0] = -1;
            so.src[0] = ts.src[t];
        }
        out->has_strfn = 1;
    }
    return compile_decimals(ctx, p, out);
}

int expr_raise(tgpu_ctx* ctx, int64_t errbits)
{
    if (errbits & TG_ERR_BIT_DIV_ZERO) return tg_fail(ctx, TGPU_ERR_DIVISION_BY_ZERO, "Division by zero");
    if (errbits & TG_ERR_BIT_OVERFLOW) return tg_fail(ctx, TGPU_ERR_NUMERIC_VALUE_OUT_OF_RANGE, "bigint arithmetic overflow");
    if (errbits & TG_ERR_BIT_DECIMAL_OVERFLOW) return tg_fail(ctx, TGPU_ERR_NUMERIC_VALUE_OUT_OF_RANGE, "Decimal overflow");
    if (errbits & TG_ERR_BIT_INVALID_CAST) return tg_fail(ctx, TGPU_ERR_INVALID_CAST_ARGUMENT, "Unable to cast double to bigint");
    if (errbits & TG_ERR_BIT_CONCAT_TOO_LARGE) return tg_fail(ctx, TGPU_ERR_INVALID_FUNCTION_ARGUMENT, "Concatenated string is too large");
    return TGPU_OK;
}

// ---- NVRTC code generation of programs -------------------------------------------------------------------------------
void fp_appendf(std::string& s, const char* fmt, ...)
{
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    s += buf;
}

static std::string fp_operand(const DOperand& o)
{
    char buf[128];
    switch (o.kind) {
        case TGPU_OPND_COLUMN: snprintf(buf, sizeof(buf), "Value{c%d, c%dn}", o.index, o.index); break;
        case TGPU_OPND_TEMP: snprintf(buf, sizeof(buf), "Value{t%d, tn%d}", o.index, o.index); break;
        case TGPU_OPND_CONST: snprintf(buf, sizeof(buf), "Value{(long long)0x%llxULL, false}", (unsigned long long)o.imm); break;
        default: snprintf(buf, sizeof(buf), "Value{0, true}"); break;
    }
    return buf;
}

// the error operand o carries (see vm_error): a temp's, never a column's or a constant's
static std::string fp_operand_error(const DOperand& o)
{
    return o.kind == TGPU_OPND_TEMP ? "te" + std::to_string(o.index) : "0u";
}

// a VARCHAR operand of generated code: its NULL flag and its StrRef (channel k: locals c<k>n / s<k>; constants: the tg_pool array)
static void fp_str_operand(const DProgram& prog, const DOperand& o, std::string* isnull, std::string* ref)
{
    char buf[160];
    if (o.kind == TGPU_OPND_COLUMN) {
        snprintf(buf, sizeof(buf), "c%dn", o.index); *isnull = buf;
        snprintf(buf, sizeof(buf), "s%d", o.index); *ref = buf;
    }
    else if (o.kind == TGPU_OPND_CONST) {
        *isnull = "false";
        snprintf(buf, sizeof(buf), "StrRef{(const uint8_t*)tg_pool + %d, %d}", prog.str_off[o.imm], prog.str_len[o.imm]);
        *ref = buf;
    }
    else if (o.kind == TGPU_OPND_TEMP) {
        snprintf(buf, sizeof(buf), "tn%d", o.index); *isnull = buf;
        snprintf(buf, sizeof(buf), "v%d", o.index); *ref = buf;
    }
    else { *isnull = "true"; *ref = "StrRef{nullptr, 0}"; }
}

// the first byte of a VARCHAR source in generated code (see DCat): the channel's byte buffer or the constant in tg_pool; `ref` for none
static std::string fp_src_base(const DProgram& prog, int32_t src, const std::string& ref)
{
    if (src == TGD_SRC_NONE) return ref + ".p";
    if (src >= 0) return "strs.bytes[" + std::to_string(prog.str_slot[src]) + "]";
    return "((const uint8_t*)tg_pool + " + std::to_string(prog.str_off[-(src + 1)]) + ")";
}

// straight-line code of one string function: LENGTH (BIGINT t<d>), the views SUBSTR and the trims write (StrRef v<d>), CONCAT (its total
// length in t<d>, its new pieces in StrRef q<slot>).  Errors as vm_step_str.
static void fp_emit_strfn_insn(std::string& s, const DProgram& prog, int i)
{
    const DInsn& in = prog.insns[i];
    const int d = in.dst;
    std::string an, a, bn, b;
    fp_str_operand(prog, in.a, &an, &a);
    const std::string ea = fp_operand_error(in.a);
    if (in.op == TGPU_EX_CONCAT) {
        const DCat& k = prog.cat[i];
        fp_str_operand(prog, in.b, &bn, &b);
        fp_appendf(s, "    { const bool an = %s, bn = %s; const bool rn = an || bn; long long tot = 0;\n", an.c_str(), bn.c_str());
        if (k.a_slot >= 0 || k.b_slot >= 0) {
            s += "      if (!rn) {";
            if (k.a_slot >= 0) fp_appendf(s, " q%d = %s;", k.a_slot, a.c_str());
            if (k.b_slot >= 0) fp_appendf(s, " q%d = %s;", k.b_slot, b.c_str());
            s += " }\n";
        }
        s += "      if (!rn) tot = 0";
        for (int q = 0; q < k.n; q++) fp_appendf(s, " + (long long)q%d.len", k.slot[q]);
        s += ";\n";
        fp_appendf(s, "      t%d = tot; tn%d = rn; te%d = vm_error_call(an, %s, bn, %s, 0u, rn, %s); }\n", d, d, d, ea.c_str(), fp_operand_error(in.b).c_str(),
                   k.inner ? "0u" : "tot > TGD_MAX_CONCAT_BYTES ? (unsigned int)TG_ERR_BIT_CONCAT_TOO_LARGE : 0u");
        return;
    }
    fp_appendf(s, "    { const bool an = %s; const StrRef a = %s;\n", an.c_str(), a.c_str());
    switch (in.op) {
        case TGPU_EX_LENGTH:
            fp_appendf(s, "      t%d = an ? 0LL : tg_utf8_count(a); tn%d = an; te%d = %s; }\n", d, d, d, ea.c_str());
            break;
        case TGPU_EX_SUBSTR: {
            const bool has_len = in.c.kind != TGPU_OPND_NONE;
            fp_appendf(s, "      const Value b = %s, c = %s; const bool rn = an || b.is_null || c.is_null;\n", fp_operand(in.b).c_str(),
                       has_len ? fp_operand(in.c).c_str() : "Value{0, false}");
            fp_appendf(s, "      te%d = vm_error_call(an, %s, b.is_null, %s, %s, rn, 0u);\n", d, ea.c_str(), fp_operand_error(in.b).c_str(),
                       has_len ? fp_operand_error(in.c).c_str() : "0u");
            fp_appendf(s, "      v%d = rn ? StrRef{nullptr, 0} : tg_substr(a, b.bits, %s, c.bits); tn%d = rn; }\n", d, has_len ? "true" : "false", d);
            break;
        }
        default:
            fp_appendf(s, "      v%d = an ? StrRef{nullptr, 0} : tg_trim(a, %s, %s); tn%d = an; te%d = %s; }\n", d, in.op != TGPU_EX_RTRIM ? "true" : "false",
                       in.op != TGPU_EX_LTRIM ? "true" : "false", d, d, ea.c_str());
            break;
    }
}

// `x` (a StrRef) equals pool string k: the length decides first, then packed 8-byte words against immediates (a constant of more than
// 64 bytes is compared with the pool's copy)
static std::string fp_str_eq_const(const std::string& x, const DProgram& prog, int64_t k)
{
    const uint8_t* b = prog.str_bytes + prog.str_off[k];
    const int n = prog.str_len[k];
    std::string e = "(" + x + ".len == " + std::to_string(n);
    if (n > 64) return e + " && tg_str_eq(" + x + ", StrRef{(const uint8_t*)tg_pool + " + std::to_string(prog.str_off[k]) + ", " + std::to_string(n) + "}))";
    for (int i = 0; i < n; i += 8) {
        const int k = n - i < 8 ? n - i : 8;
        unsigned long long w = 0;
        for (int j = 0; j < k; j++) w |= (unsigned long long)b[i + j] << (8 * j);
        char buf[96];
        snprintf(buf, sizeof(buf), " && tg_ld_bytes(%s.p + %d, %d) == 0x%llxULL", x.c_str(), i, k, w);
        e += buf;
    }
    return e + ")";
}

// straight-line code of one instruction over VARCHAR operands (result BOOLEAN, never an error)
static void fp_emit_str_insn(std::string& s, const DProgram& prog, const DInsn& in)
{
    if (string_function(in.op)) {
        fp_emit_strfn_insn(s, prog, (int)(&in - prog.insns));
        return;
    }
    std::string an, a, bn, b, cn, c;
    fp_str_operand(prog, in.a, &an, &a);
    fp_appendf(s, "    { const bool an = %s; const StrRef a = %s; bool r = false, rn = an;\n", an.c_str(), a.c_str());
    switch (in.op) {
        case TGPU_EX_IS_NULL: s += "      r = an; rn = false;\n"; break;
        case TGPU_EX_IS_NOT_NULL: s += "      r = !an; rn = false;\n"; break;
        case TGPU_EX_LIKE: fp_appendf(s, "      if (!an) r = tg_like_%d(a);\n", (int)in.b.imm); break;
        case TGPU_EX_IN: {
            const int li = (int)in.b.imm;
            s += "      if (!an) r = false";
            for (int k = 0; k < prog.in_count[li]; k++) {
                const int64_t si = prog.in_values[prog.in_offset[li] + k];
                s += "\n        || " + fp_str_eq_const("a", prog, si);
            }
            s += ";\n";
            break;
        }
        case TGPU_EX_BETWEEN:
            fp_str_operand(prog, in.b, &bn, &b);
            fp_str_operand(prog, in.c, &cn, &c);
            fp_appendf(s, "      { const bool n1 = an || %s, n2 = an || %s; const bool f1 = !n1 && tg_str_cmp(a, %s) < 0, f2 = !n2 && tg_str_cmp(a, %s) > 0;\n",
                       bn.c_str(), cn.c_str(), b.c_str(), c.c_str());
            s += "        rn = !(f1 || f2) && (n1 || n2); r = !(f1 || f2 || rn); }\n";
            break;
        default:
            fp_str_operand(prog, in.b, &bn, &b);
            fp_appendf(s, "      rn = an || %s;\n", bn.c_str());
            if ((in.op == TGPU_EX_EQ || in.op == TGPU_EX_NE) && in.b.kind == TGPU_OPND_CONST)
                s += std::string("      if (!rn) r = ") + (in.op == TGPU_EX_NE ? "!" : "") + fp_str_eq_const("a", prog, in.b.imm) + ";\n";
            else fp_appendf(s, "      if (!rn) r = tg_str_cmp_op(%d, a, %s);\n", in.op, b.c_str());
            break;
    }
    // the error a view temp operand carries (vm_error_str_pred); none without temp operands
    std::string e = "0u";
    if (in.a.kind == TGPU_OPND_TEMP || in.b.kind == TGPU_OPND_TEMP || in.c.kind == TGPU_OPND_TEMP) {
        const std::string ea = fp_operand_error(in.a), eb = fp_operand_error(in.b), ec = fp_operand_error(in.c);
        if (in.op == TGPU_EX_IS_NULL || in.op == TGPU_EX_IS_NOT_NULL || in.op == TGPU_EX_LIKE || in.op == TGPU_EX_IN) e = ea;
        else if (in.op == TGPU_EX_BETWEEN) {
            fp_str_operand(prog, in.b, &bn, &b);
            e = "((" + ea + ") || an ? (" + ea + ") : (" + eb + ") ? (" + eb + ") : (!(" + bn + ") && tg_str_cmp(" + b + ", a) > 0) ? 0u : (" + ec + "))";
        }
        else e = "((" + ea + ") || an ? (" + ea + ") : (" + eb + "))";
    }
    fp_appendf(s, "      t%d = r ? 1 : 0; tn%d = rn; te%d = %s; }\n", in.dst, in.dst, in.dst, e.c_str());
}

// module-scope data and functions the string operations of `prog` use: the constant pool and one matcher per LIKE pattern, whose
// length bounds, prefix and suffix are immediates; the middle runs the shared matcher over the compiled pattern
static std::string fp_string_decls(const DProgram& prog)
{
    std::string s;
    if (prog.num_strings > 0) {
        int words = 0;
        for (int k = 0; k < prog.num_strings; k++) words = std::max(words, (prog.str_off[k] + prog.str_len[k] + 7) / 8);
        s += "__device__ const unsigned long long tg_pool[" + std::to_string(std::max(words, 1)) + "] = {";
        for (int w = 0; w < std::max(words, 1); w++) {
            unsigned long long v = 0;
            for (int j = 0; j < 8 && w * 8 + j < TGPU_MAX_STRING_BYTES; j++) v |= (unsigned long long)prog.str_bytes[w * 8 + j] << (8 * j);
            fp_appendf(s, "%s0x%llxULL", w ? "," : "", v);
        }
        s += "};\n";
    }
    for (int k = 0; k < prog.num_likes; k++) {
        const DLike& L = prog.likes[k];
        if (L.kind != TGD_LIKE_NONE) {
            fp_appendf(s, "__device__ const unsigned long long tg_like_data_%d[%d] = {", k, (int)(sizeof(DLike) / 8));
            const unsigned long long* raw = (const unsigned long long*)&L;
            for (size_t w = 0; w < sizeof(DLike) / 8; w++) fp_appendf(s, "%s0x%llxULL", w ? "," : "", raw[w]);
            s += "};\n";
        }
        fp_appendf(s, "__device__ __forceinline__ bool tg_like_%d(StrRef s) {\n  if (s.len < %d) return false;\n", k, L.min_size);
        if (L.max_size >= 0) fp_appendf(s, "  if (s.len > %d) return false;\n", L.max_size);
        for (int i = 0; i < L.prefix_len; i += 8) {
            const int n = std::min(8, L.prefix_len - i);
            unsigned long long w = 0;
            for (int j = 0; j < n; j++) w |= (unsigned long long)L.bytes[i + j] << (8 * j);
            fp_appendf(s, "  if (tg_ld_bytes(s.p + %d, %d) != 0x%llxULL) return false;\n", i, n, w);
        }
        for (int i = 0; i < L.suffix_len; i += 8) {
            const int n = std::min(8, L.suffix_len - i);
            unsigned long long w = 0;
            for (int j = 0; j < n; j++) w |= (unsigned long long)L.bytes[L.prefix_len + i + j] << (8 * j);
            fp_appendf(s, "  if (tg_ld_bytes(s.p + s.len - %d, %d) != 0x%llxULL) return false;\n", L.suffix_len - i, n, w);
        }
        if (L.kind == TGD_LIKE_NONE) s += "  return true;\n}\n";
        else fp_appendf(s, "  return %s(*(const DLike*)tg_like_data_%d, s.p + %d, s.len - %d);\n}\n",
                        L.kind == TGD_LIKE_FJS ? "tg_like_fjs" : L.kind == TGD_LIKE_DFA ? "tg_like_dfa" : "tg_like_nfa", k, L.prefix_len,
                        L.prefix_len + L.suffix_len);
    }
    return s;
}

// a DECIMAL operand of generated code as a DVal (`lng`: a long decimal: locals ch<k> / th<i> hold the high words)
static std::string fp_dec_operand(const DOperand& o, bool lng, long long khi)
{
    char buf[160];
    switch (o.kind) {
        case TGPU_OPND_COLUMN:
            if (lng) snprintf(buf, sizeof(buf), "DVal{U128{(unsigned long long)ch%d, (unsigned long long)c%d}, c%dn}", o.index, o.index, o.index);
            else snprintf(buf, sizeof(buf), "DVal{u128_sx(c%d), c%dn}", o.index, o.index);
            break;
        case TGPU_OPND_TEMP:
            if (lng) snprintf(buf, sizeof(buf), "DVal{U128{(unsigned long long)th%d, (unsigned long long)t%d}, tn%d}", o.index, o.index, o.index);
            else snprintf(buf, sizeof(buf), "DVal{u128_sx(t%d), tn%d}", o.index, o.index);
            break;
        case TGPU_OPND_CONST:
            snprintf(buf, sizeof(buf), "DVal{U128{0x%llxULL, 0x%llxULL}, false}", lng ? (unsigned long long)khi : (unsigned long long)(o.imm >> 63),
                     (unsigned long long)o.imm);
            break;
        default: snprintf(buf, sizeof(buf), "DVal{U128{0ULL, 0ULL}, true}"); break;
    }
    return buf;
}

// straight-line code of one DECIMAL instruction: vm_apply_dec with the instruction's method as constants, so that the compiler keeps only
// that method's path (a short one stays 64-bit code with 10^k as immediates); the high word is kept for long results only
static void fp_emit_dec_insn(std::string& s, const DProgram& prog, int i)
{
    const DInsn& in = prog.insns[i];
    const DDec& d = prog.dec[i];
    const bool long_dst = (prog.long_temps >> in.dst) & 1;
    if (in.op == TGPU_EX_IN) {
        const int li = (int)in.b.imm;
        fp_appendf(s, "    { DVal a = %s; bool hit = false;\n", fp_dec_operand(in.a, d.la, 0).c_str());
        for (int k = 0; k < prog.in_count[li]; k++) {
            const int at = prog.in_offset[li] + k;
            const unsigned long long lo = (unsigned long long)prog.in_values[at], hi = d.la ? (unsigned long long)prog.in_hi[at] : (unsigned long long)(prog.in_values[at] >> 63);
            fp_appendf(s, "      hit |= a.v.hi == 0x%llxULL && a.v.lo == 0x%llxULL;\n", hi, lo);
        }
        fp_appendf(s, "      t%d = hit ? 1 : 0; tn%d = a.is_null; te%d = %s;%s }\n", in.dst, in.dst, in.dst, fp_operand_error(in.a).c_str(),
                   long_dst ? (" th" + std::to_string(in.dst) + " = 0;").c_str() : "");
        return;
    }
    fp_appendf(s, "    { DVal a = %s, b = %s, c = %s; unsigned int e = 0;\n", fp_dec_operand(in.a, d.la, d.hi[0]).c_str(), fp_dec_operand(in.b, d.lb, d.hi[1]).c_str(),
               fp_dec_operand(in.c, d.lc, d.hi[2]).c_str());
    fp_appendf(s, "      const DDec dd = {1, %d, %d, %d, %d, 0, 0, 0, %d, %d, %d, 0, %lldLL, %lldLL, {0, 0, 0}};\n", d.la, d.lb, d.lc, d.lr, d.k0, d.k1, d.k2,
               d.m0, d.m1);
    fp_appendf(s, "      DVal x = vm_apply_dec(%d, %d, dd, a, b, c, &e);\n", in.op, in.vtype);
    fp_appendf(s, "      e = vm_error_dec(%d, a, %s, b, %s, %s, e); t%d = (long long)x.v.lo; tn%d = x.is_null; te%d = e;", in.op, fp_operand_error(in.a).c_str(),
               fp_operand_error(in.b).c_str(), fp_operand_error(in.c).c_str(), in.dst, in.dst, in.dst);
    if (long_dst) fp_appendf(s, " th%d = (long long)x.v.hi;", in.dst);
    s += " }\n";
}

void fp_emit_insns(std::string& s, const DProgram& prog, int first, int last)
{
    for (int i = first; i < last; i++) {
        const DInsn& in = prog.insns[i];
        if (prog.has_dec && prog.dec[i].is_dec) fp_emit_dec_insn(s, prog, i);
        else if (in.vtype == TGPU_V_VARCHAR) fp_emit_str_insn(s, prog, in);
        else if (in.op == TGPU_EX_IN) {
            int li = (int)in.b.imm;
            fp_appendf(s, "    { Value a = %s; bool hit = false;\n", fp_operand(in.a).c_str());
            for (int k = 0; k < prog.in_count[li]; k++) {
                unsigned long long c = (unsigned long long)prog.in_values[prog.in_offset[li] + k];
                if (in.vtype == TGPU_V_DOUBLE) fp_appendf(s, "      hit |= __longlong_as_double(a.bits) == __longlong_as_double((long long)0x%llxULL);\n", c);
                else fp_appendf(s, "      hit |= a.bits == (long long)0x%llxULL;\n", c);
            }
            fp_appendf(s, "      t%d = hit ? 1 : 0; tn%d = a.is_null; te%d = %s; }\n", in.dst, in.dst, in.dst, fp_operand_error(in.a).c_str());
        }
        else {
            // operands are read into locals first: dst may be one of them, and vm_error needs their values
            fp_appendf(s, "    { Value a = %s, b = %s, c = %s; unsigned int e = 0; Value x = vm_apply(%d, %d, a, b, c, &e);\n", fp_operand(in.a).c_str(),
                       fp_operand(in.b).c_str(), fp_operand(in.c).c_str(), in.op, in.vtype);
            fp_appendf(s, "      e = vm_error(%d, %d, a, %s, b, %s, c, %s, e); t%d = x.bits; tn%d = x.is_null; te%d = e; }\n", in.op, in.vtype,
                       fp_operand_error(in.a).c_str(), fp_operand_error(in.b).c_str(), fp_operand_error(in.c).c_str(), in.dst, in.dst, in.dst);
        }
    }
}

void fp_emit_temps(std::string& s, const DProgram& prog)
{
    for (int t = 0; t < TGPU_MAX_TEMPS; t++) fp_appendf(s, "    long long t%d = 0; bool tn%d = true; unsigned int te%d = 0;\n", t, t, t);
    // high words of the temps that hold a long DECIMAL
    for (int t = 0; t < TGPU_MAX_TEMPS; t++)
        if ((prog.long_temps >> t) & 1) fp_appendf(s, "    long long th%d = 0;\n", t);
    // string functions: the views temps hold and the captured concatenation pieces
    if (prog.has_strfn) {
        for (int t = 0; t < TGPU_MAX_TEMPS; t++) fp_appendf(s, "    StrRef v%d = {nullptr, 0};\n", t);
        for (int q = 0; q < prog.num_piece_slots; q++) fp_appendf(s, "    StrRef q%d = {nullptr, 0};\n", q);
    }
}

void fp_mark_columns(const DProgram& prog, int first, int last, bool* used)
{
    for (int i = first; i < last; i++) {
        const DOperand* ops[3] = {&prog.insns[i].a, &prog.insns[i].b, &prog.insns[i].c};
        for (auto* o : ops)
            if (o->kind == TGPU_OPND_COLUMN) used[o->index] = true;
    }
}

}  // namespace tg

namespace {

using namespace tg;

constexpr int FP_THREADS = 256;

// ---- NVRTC specialisation of the two PageProcessor kernels ----------------------------------------------------------

// filter pass: one row per thread, writes 1/0 selection flags.  DEC: the program holds DECIMAL operations, whose temps keep a high word
// in a second shared lane (programs without DECIMAL keep the shared memory and occupancy they had)
template <bool DEC>
__global__ void __launch_bounds__(FP_THREADS) fp_filter_kernel(const DProgram* __restrict__ prog, DColumns cols, StrCols strs, int64_t n, uint8_t* __restrict__ flags,
                                                              unsigned int* __restrict__ err_out)
{
    __shared__ int64_t temps[TGPU_MAX_TEMPS * FP_THREADS];
    __shared__ int64_t temps_hi[DEC ? TGPU_MAX_TEMPS * FP_THREADS : 1];
    int64_t pieces[TGD_MAX_PIECE_SLOTS];
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    uint32_t err = 0;
    for (; i < n; i += stride) {
        uint32_t te = 0;
        uint32_t nb = vm_run<true, DEC>(prog, 0, prog->num_filter_insns, cols, i, temps + threadIdx.x, FP_THREADS, 0, &te, 0, 0, &strs,
                                        DEC ? temps_hi + threadIdx.x : nullptr, pieces);
        int ft = prog->filter_temp;
        err |= vm_temp_error(te, ft);
        bool sel = !((nb >> ft) & 1) && temps[ft * FP_THREADS + threadIdx.x] != 0;
        flags[i] = sel ? 1 : 0;
    }
    if (err) atomicOr(err_out, err);
}

// projection pass: output row j <- input row sel[j] (sel == nullptr: identity)
template <bool DEC>
__global__ void __launch_bounds__(FP_THREADS) fp_project_kernel(const DProgram* __restrict__ prog, DColumns cols, StrCols strs, const int32_t* __restrict__ sel, int64_t m,
                                                               OutCols out, unsigned int* __restrict__ err_out, unsigned int* __restrict__ any_null)
{
    __shared__ int64_t temps[TGPU_MAX_TEMPS * FP_THREADS];
    __shared__ int64_t temps_hi[DEC ? TGPU_MAX_TEMPS * FP_THREADS : 1];
    int64_t pieces[TGD_MAX_PIECE_SLOTS];
    int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    uint32_t err = 0, nulls_seen = 0;
    for (; j < m; j += stride) {
        int64_t row = sel ? sel[j] : j;
        int64_t* t = temps + threadIdx.x;
        int64_t* th = DEC ? temps_hi + threadIdx.x : nullptr;
        uint32_t te = 0;
        uint32_t nb = vm_run<true, DEC>(prog, 0, prog->num_insns, cols, row, t, FP_THREADS, 0, &te, 0, 0, &strs, th, pieces);
        // VARCHAR projections: the view in the temp or the concatenation's pieces, as (begin - source base, length) descriptors
        for (int k = 0; k < out.str_count; k++) {
            const DStrOut& so = prog->str_out[k];
            const bool isn = (nb >> so.temp) & 1;
            err |= vm_temp_error(te, so.temp);
            int2* d = (int2*)out.str_desc[k] + j * so.n;
            for (int q = 0; q < so.n; q++) {
                const int64_t v = so.slot[q] < 0 ? t[so.temp * FP_THREADS] : pieces[so.slot[q]];
                d[q] = isn ? make_int2(0, 0) : make_int2((int)(uint32_t)v, (int)(v >> 32));
            }
            out.str_nullmap[k][j] = isn ? 1 : 0;
        }
        for (int c = 0; c < out.count; c++) {
            int tp = out.temp[c];
            err |= vm_temp_error(te, tp);
            bool isn = (nb >> tp) & 1;
            int64_t v = isn ? 0 : t[tp * FP_THREADS];
            if (DEC && out.vtype[c] == TGD_V_DECIMAL_LONG) {
                ((int64_t*)out.data[c])[2 * j] = isn ? 0 : th[tp * FP_THREADS];
                ((int64_t*)out.data[c])[2 * j + 1] = v;
            }
            else if (out.vtype[c] == TGPU_V_BOOLEAN) ((int8_t*)out.data[c])[j] = (int8_t)v;
            else ((int64_t*)out.data[c])[j] = v;
            out.nullmap[c][j] = isn ? 1 : 0;
            if (isn) nulls_seen |= 1u << c;
        }
    }
    if (err) atomicOr(err_out, err);
    if (nulls_seen) atomicOr(any_null, nulls_seen);
}


// straight-line typed code for one program over channels of the given element sizes
static std::string gen_fp_source(const DProgram& prog, const int* elems, int num_channels, uint32_t nullable_mask, const std::vector<int>& pass_channels)
{
    std::string s = fp_string_decls(prog);
    bool used[TGPU_MAX_CHANNELS] = {false}, str_used[TGPU_MAX_CHANNELS] = {false};     // read as a number / as a string
    bool wide_used[TGPU_MAX_CHANNELS] = {false};                                      // read as a long DECIMAL
    for (int i = 0; i < prog.num_insns; i++) {
        const DOperand* ops[3] = {&prog.insns[i].a, &prog.insns[i].b, &prog.insns[i].c};
        const DDec& d = prog.dec[i];
        const bool lng[3] = {d.la != 0, d.lb != 0, d.lc != 0};
        for (int k = 0; k < 3; k++) {
            // substr's start and length are BIGINT operands
            const bool str = prog.insns[i].vtype == TGPU_V_VARCHAR && !(prog.insns[i].op == TGPU_EX_SUBSTR && k > 0);
            if (ops[k]->kind == TGPU_OPND_COLUMN) (str ? str_used : lng[k] ? wide_used : used)[ops[k]->index] = true;
        }
    }
    std::string loads, temps;
    for (int c = 0; c < num_channels && c < TGPU_MAX_CHANNELS; c++) {
        if (!used[c] && !str_used[c] && !wide_used[c]) continue;
        if (wide_used[c])
            fp_appendf(loads, "    const longlong2 c%dw = ((const longlong2*)cols.cols[%d].data)[row]; const long long ch%d = c%dw.x, c%d = c%dw.y;", c, c, c, c, c, c);
        else if (used[c]) fp_appendf(loads, "    const long long c%d = tg_load_elem<%d>(cols.cols[%d].data, row);", c, elems[c], c);
        if ((nullable_mask >> c) & 1) fp_appendf(loads, " const bool c%dn = !tg_valid(cols.cols[%d].validity, row);\n", c, c);
        else fp_appendf(loads, " const bool c%dn = false;\n", c);
        if (str_used[c]) fp_appendf(loads, "    const StrRef s%d = tg_str(strs, %d, row);\n", c, prog.str_slot[c]);
    }
    fp_emit_temps(temps, prog);
    const bool wide_out = prog.long_temps != 0;
    // value, NULL flag and carried error of the temp behind each computed output column (the only errors a projection raises)
    std::string output_switch = "    for (int c = 0; c < out.count; c++) {\n      long long v = 0; bool isn = true; unsigned int e = 0;\n";
    if (wide_out) output_switch += "      long long hv = 0;\n";
    output_switch += "      switch (out.temp[c]) {\n";
    for (int t = 0; t < TGPU_MAX_TEMPS; t++) {
        if ((prog.long_temps >> t) & 1) fp_appendf(output_switch, "        case %d: v = t%d; hv = th%d; isn = tn%d; e = te%d; break;\n", t, t, t, t, t);
        else fp_appendf(output_switch, "        case %d: v = t%d; isn = tn%d; e = te%d; break;\n", t, t, t, t);
    }
    output_switch += "      }\n      err |= e;\n      if (isn) v = 0;\n";
    // the store of one computed output cell: a long DECIMAL writes a 16-byte (high, low) cell
    std::string store = "      if (out.vtype[c] == TGD_V_BOOLEAN) ((signed char*)out.data[c])[j] = (signed char)v; else ((long long*)out.data[c])[j] = v;\n";
    if (wide_out)
        store = "      if (isn) hv = 0;\n      if (out.vtype[c] == TGD_V_DECIMAL_LONG) ((longlong2*)out.data[c])[j] = make_longlong2(hv, v);\n"
                "      else if (out.vtype[c] == TGD_V_BOOLEAN) ((signed char*)out.data[c])[j] = (signed char)v; else ((long long*)out.data[c])[j] = v;\n";
    // VARCHAR projections: one (begin, length) descriptor per piece into the piece's source, and the NULL byte
    std::string str_store;
    for (int k = 0; k < prog.num_str_outs; k++) {
        const DStrOut& so = prog.str_out[k];
        fp_appendf(str_store, "    { const bool isn = tn%d; err |= te%d; int2* d = (int2*)out.str_desc[%d] + j * %d;\n", so.temp, so.temp, k, so.n);
        for (int q = 0; q < so.n; q++) {
            const std::string ref = so.slot[q] < 0 ? "v" + std::to_string(so.temp) : "q" + std::to_string(so.slot[q]);
            fp_appendf(str_store, "      d[%d] = isn ? make_int2(0, 0) : make_int2((int)(%s.p - %s), %s.len);\n", q, ref.c_str(),
                       fp_src_base(prog, so.src[q], ref).c_str(), ref.c_str());
        }
        fp_appendf(str_store, "      out.str_nullmap[%d][j] = isn ? 1 : 0; }\n", k);
    }
    // filter kernel
    s += "extern \"C\" __global__ void __launch_bounds__(256) tg_fp_filter_jit(DColumns cols, StrCols strs, long long n, unsigned char* flags, unsigned int* err_out) {\n";
    s += "  unsigned int err = 0;\n  long long stride = (long long)gridDim.x * blockDim.x;\n";
    s += "  for (long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x; row < n; row += stride) {\n";
    s += loads + temps;
    fp_emit_insns(s, prog, 0, prog.num_filter_insns);
    if (prog.filter_temp >= 0) fp_appendf(s, "    err |= te%d;\n    flags[row] = (!tn%d && t%d != 0) ? 1 : 0;\n", prog.filter_temp, prog.filter_temp, prog.filter_temp);
    else s += "    flags[row] = 1;\n";
    s += "  }\n  if (err) atomicOr(err_out, err);\n}\n";
    // projection kernel
    s += "extern \"C\" __global__ void __launch_bounds__(256) tg_fp_project_jit(DColumns cols, StrCols strs, const int* sel, long long m, OutCols out, unsigned int* err_out, unsigned int* any_null) {\n";
    s += "  unsigned int err = 0, nulls_seen = 0;\n  long long stride = (long long)gridDim.x * blockDim.x;\n";
    s += "  for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < m; j += stride) {\n";
    s += "    const long long row = sel ? sel[j] : j;\n";
    s += loads + temps;
    fp_emit_insns(s, prog, 0, prog.num_insns);
    s += output_switch;
    s += store;
    s += "      out.nullmap[c][j] = isn ? 1 : 0;\n      if (isn) nulls_seen |= 1u << c;\n    }\n";
    s += str_store;
    s += "  }\n  if (err) atomicOr(err_out, err);\n  if (nulls_seen) atomicOr(any_null, nulls_seen);\n}\n";
    // chunked two-pass form (no selection vector): per-row functors + the two kernels around the bodies of device_lib.cuh
    bool chunkable = prog.filter_temp >= 0;
    for (int ch : pass_channels)
        if (ch < 0 || ch >= num_channels || elems[ch] == 0) chunkable = false;     // variable-width pass-through: not in this form
    if (!chunkable) return s;
    s += "struct FProg {\n";
    s += "  static __device__ __forceinline__ bool filter(const DColumns& cols, const StrCols& strs, long long row, unsigned int* errp) {\n    unsigned int err = 0;\n";
    s += loads + temps;
    fp_emit_insns(s, prog, 0, prog.num_filter_insns);
    fp_appendf(s, "    err |= te%d;\n    *errp |= err;\n    return !tn%d && t%d != 0;\n  }\n", prog.filter_temp, prog.filter_temp, prog.filter_temp);
    s += "  static __device__ __forceinline__ void row(const DColumns& cols, const StrCols& strs, long long row, long long j, const OutCols& out, unsigned int* errp, unsigned int* nullsp) {\n";
    s += "    unsigned int err = 0, nulls_seen = 0;\n";
    s += loads + temps;
    fp_emit_insns(s, prog, 0, prog.num_insns);
    s += output_switch;
    s += store;
    s += "      out.nullmap[c][j] = isn ? 1 : 0;\n      if (isn) nulls_seen |= 1u << c;\n    }\n";
    s += str_store;
    for (size_t k = 0; k < pass_channels.size(); k++) {
        int ch = pass_channels[k];
        const char* ty = elems[ch] == 16 ? "int4" : elems[ch] == 8 ? "long long" : elems[ch] == 4 ? "int" : elems[ch] == 2 ? "short" : "signed char";
        fp_appendf(s, "    ((%s*)out.pass_data[%d])[j] = ((const %s*)cols.cols[%d].data)[row];\n", ty, (int)k, ty, ch);
        if ((nullable_mask >> ch) & 1) fp_appendf(s, "    out.pass_nullmap[%d][j] = tg_valid(cols.cols[%d].validity, row) ? 0 : 1;\n", (int)k, ch);
    }
    s += "    *errp |= err;\n    *nullsp |= nulls_seen;\n  }\n};\n";
    s += "extern \"C\" __global__ void __launch_bounds__(256) tg_fp_filter_chunks_jit(DColumns cols, StrCols strs, long long n, long long chunk, unsigned char* flags, "
         "unsigned int* counts, unsigned int* err_out) { fp_filter_chunks_body<FProg>(cols, strs, n, chunk, flags, counts, err_out); }\n";
    s += "extern \"C\" __global__ void __launch_bounds__(256) tg_fp_project_chunks_jit(DColumns cols, StrCols strs, const unsigned char* flags, long long n, long long chunk, "
         "const long long* chunk_off, OutCols out, unsigned int* err_out, unsigned int* any_null) "
         "{ fp_project_chunks_body<FProg>(cols, strs, flags, n, chunk, chunk_off, out, err_out, any_null); }\n";
    return s;
}

// exclusive scan of the chunk counts of the chunked FilterAndProject form (one CTA)
__global__ void __launch_bounds__(256) fp_chunk_scan_kernel(const unsigned int* __restrict__ counts, int chunks, long long* __restrict__ chunk_off,
                                                            long long* __restrict__ total)
{
    __shared__ long long part[256];
    const int t = threadIdx.x;
    const int per = (chunks + 255) / 256;
    const int b0 = min(chunks, t * per), b1 = min(chunks, b0 + per);
    long long sum = 0;
    for (int b = b0; b < b1; b++) sum += counts[b];
    part[t] = sum;
    __syncthreads();
    for (int off = 1; off < 256; off <<= 1) {
        long long v = t >= off ? part[t - off] : 0;
        __syncthreads();
        part[t] += v;
        __syncthreads();
    }
    long long run = part[t] - sum;
    for (int b = b0; b < b1; b++) {
        chunk_off[b] = run;
        run += counts[b];
    }
    if (t == 255) *total = part[255];
}

// ---- VARCHAR projection columns ------------------------------------------------------------------------------------------------
// row length = the sum of the row's piece lengths (0 for a NULL row); len[m] = 0 so that the exclusive scan ends in the total
__global__ void __launch_bounds__(256) fp_str_lengths_kernel(const int2* __restrict__ desc, int np, const uint8_t* __restrict__ nullmap, int64_t m,
                                                            long long* __restrict__ len, unsigned int* __restrict__ any_null)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    unsigned int seen = 0;
    for (; i < m; i += stride) {
        long long l = 0;
        for (int q = 0; q < np; q++) l += desc[i * np + q].y;
        len[i] = l;
        seen |= nullmap[i];
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) len[m] = 0;
    if (seen) atomicOr(any_null, 1u);
}

__global__ void __launch_bounds__(256) fp_str_narrow_kernel(const long long* __restrict__ off64, int64_t n, int32_t* __restrict__ off)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) off[i] = (int32_t)off64[i];
}

// the sources of one VARCHAR projection's pieces
struct StrSrcs {
    const uint8_t* base[TGD_MAX_PIECES];
};

constexpr int FPS_WARPS = 8;      // warps per CTA of the assembly kernel; a warp owns 32 consecutive output rows at a time

// Byte assembly: a warp owns the contiguous destination range of 32 consecutive output rows.  Its lanes note where each (row, piece)
// segment starts in the destination and in its source, then store the range as aligned 8-byte words: a lane finds the segment of its
// word's first byte by binary search and reads the word's bytes with at most one aligned-word load pair per segment it crosses.  Words
// shared with the neighbouring tiles are stored byte by byte.
__global__ void __launch_bounds__(FPS_WARPS * 32) fp_str_assemble_kernel(const int2* __restrict__ desc, int np, StrSrcs srcs, const int32_t* __restrict__ off,
                                                                        int64_t m, uint8_t* __restrict__ dst)
{
    __shared__ int32_t seg_dst[FPS_WARPS][32 * TGD_MAX_PIECES + 1];
    __shared__ int32_t seg_src[FPS_WARPS][32 * TGD_MAX_PIECES];
    __shared__ const uint8_t* base[TGD_MAX_PIECES];
#pragma unroll
    for (int q = 0; q < TGD_MAX_PIECES; q++)      // constant indices: the parameter is read in place, not copied to the stack
        if (threadIdx.x == q) base[q] = srcs.base[q];
    __syncthreads();
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int32_t* sd = seg_dst[w];
    int32_t* ss = seg_src[w];
    const int nseg = 32 * np;
    const int64_t tiles = (m + 31) / 32;
    for (int64_t tile = (int64_t)blockIdx.x * FPS_WARPS + w; tile < tiles; tile += (int64_t)gridDim.x * FPS_WARPS) {
        const int64_t r0 = tile * 32;
        const int64_t r = r0 + lane;
        const int32_t t1 = off[r0 + 32 < m ? r0 + 32 : m];
        int32_t d = r < m ? off[r] : t1;
        for (int q = 0; q < np; q++) {
            const int2 x = r < m ? desc[r * np + q] : make_int2(0, 0);
            sd[lane * np + q] = d;
            ss[lane * np + q] = x.x;
            d += x.y;
        }
        if (lane == 0) sd[nseg] = t1;
        __syncwarp();
        const int32_t t0 = sd[0];
        if (t1 > t0) {
            for (int64_t word = (t0 >> 3) + lane; word <= (int64_t)((t1 - 1) >> 3); word += 32) {
                const int32_t wb = (int32_t)(word * 8);
                const int32_t b0 = wb > t0 ? wb : t0, b1 = wb + 8 < t1 ? wb + 8 : t1;
                // the last segment that starts at or before b0 holds it (empty segments share their start with the next one)
                int lo = 0, hi = nseg - 1;
                while (lo < hi) {
                    const int mid = (lo + hi + 1) >> 1;
                    if (sd[mid] <= b0) lo = mid;
                    else hi = mid - 1;
                }
                int sg = lo;
                unsigned long long v = 0;
                int32_t b = b0;
                while (b < b1) {
                    while (sd[sg + 1] <= b) sg++;
                    const int32_t e = sd[sg + 1] < b1 ? sd[sg + 1] : b1;
                    const uint8_t* src = base[sg % np] + ss[sg] + (b - sd[sg]);
                    v |= tg_ld_bytes(src, e - b) << (8 * (b - wb));
                    b = e;
                }
                if (b0 == wb && b1 == wb + 8) *(unsigned long long*)(dst + wb) = v;
                else
                    for (int32_t k = b0; k < b1; k++) dst[k] = (uint8_t)(v >> (8 * (k - wb)));
            }
        }
        __syncwarp();
    }
}

struct FilterProjectOp : tgpu_op {
    DProgram host_prog;
    DevBuf d_prog;
    std::vector<tgpu_projection> projections;
    int32_t max_channel = -1;
    StrCols cur_strs;                    // the UTF8 channels of the page in flight (sources of VARCHAR projections)
    int64_t utf8_limit = INT32_MAX;      // the most bytes a VARCHAR projection column holds (int32 offsets)
    std::vector<OwnedPage*> pending;
    size_t next_out = 0;
    bool finishing = false;

    explicit FilterProjectOp(tgpu_ctx* c) : tgpu_op(c) {}
    ~FilterProjectOp() override { for (size_t i = next_out; i < pending.size(); i++) delete pending[i]; }

    bool needs_input() override { return !finishing && next_out >= pending.size(); }

    int add_input(const tgpu_page* page) override
    {
        for (size_t i = next_out; i < pending.size(); i++) delete pending[i];   // pages the caller never took
        pending.clear();
        next_out = 0;
        int64_t n = page->num_rows;
        if (n == 0) return TGPU_OK;
        if (n > (int64_t)INT32_MAX) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "page has more than 2^31-1 positions");
        DevPage in;
        TG_TRY(tg_ingest_page(ctx, page, &in));
        if (max_channel >= (int32_t)in.cols.size()) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "program reads channel %d, page has %zu", max_channel, in.cols.size());
        DColumns cols;
        memset(&cols, 0, sizeof(cols));
        for (size_t c = 0; c < in.cols.size() && c < TGPU_MAX_CHANNELS; c++) {
            if ((int32_t)c <= max_channel && in.cols[c].type == TGPU_UTF8) {
                // only pass-through is allowed for variable-width columns; computed operands were validated below
            }
            cols.cols[c] = tg_colref(in.cols[c]);
        }
        for (int i = 0; i < host_prog.num_insns; i++) {
            const DOperand* ops[3] = {&host_prog.insns[i].a, &host_prog.insns[i].b, &host_prog.insns[i].c};
            const bool str = host_prog.insns[i].vtype == TGPU_V_VARCHAR;
            const DDec& dd = host_prog.dec[i];
            // IF's condition is BOOLEAN whatever the vtype: a BOOLEAN channel is TGPU_INT8 (a DOUBLE read as raw bits would make -0.0 TRUE)
            const bool if_cond_col = host_prog.insns[i].op == TGPU_EX_IF && ops[0]->kind == TGPU_OPND_COLUMN;
            if (if_cond_col && in.cols[ops[0]->index].type != TGPU_INT8)
                return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d reads channel %d as the BOOLEAN condition of IF, the page's channel is not INT8", i, ops[0]->index);
            if (dd.is_dec && host_prog.insns[i].vtype == TGPU_V_DECIMAL) {
                // a short DECIMAL channel is TGPU_INT64, a long one TGPU_INT128 (IF's condition, checked above, is not a DECIMAL operand)
                const bool lng[3] = {dd.la != 0, dd.lb != 0, dd.lc != 0};
                for (int k = if_cond_col ? 1 : 0; k < 3; k++) {
                    if (ops[k]->kind != TGPU_OPND_COLUMN) continue;
                    const int want = lng[k] ? TGPU_INT128 : TGPU_INT64;
                    if (in.cols[ops[k]->index].type != want)
                        return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d reads channel %d as a %s DECIMAL, the page's channel is not %s", i, ops[k]->index,
                                       lng[k] ? "long" : "short", lng[k] ? "INT128" : "INT64");
                }
                continue;
            }
            for (auto* o : ops) {
                if (o->kind != TGPU_OPND_COLUMN) continue;
                if (str && host_prog.insns[i].op == TGPU_EX_SUBSTR && o != ops[0]) {
                    // substr's start and length: an integer channel
                    const int t = in.cols[o->index].type;
                    if (t != TGPU_INT64 && t != TGPU_INT32 && t != TGPU_INT16 && t != TGPU_INT8)
                        return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d reads channel %d as BIGINT, the page's channel is not an integer", i, o->index);
                    continue;
                }
                if (str && in.cols[o->index].type != TGPU_UTF8)
                    return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d reads channel %d as VARCHAR, the page's channel is not UTF8", i, o->index);
                if (!str && (in.cols[o->index].elem_size() == 0 || in.cols[o->index].elem_size() == 16 || in.cols[o->index].type == TGPU_FLOAT32))
                    return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "expressions over variable-width / 128-bit / REAL channel %d are not supported on the GPU path", o->index);
            }
        }
        StrCols strs;
        memset(&strs, 0, sizeof(strs));
        for (int k = 0; k < host_prog.num_str_channels; k++) {
            strs.offsets[k] = in.cols[host_prog.str_channel[k]].offsets;
            strs.bytes[k] = (const uint8_t*)in.cols[host_prog.str_channel[k]].data;
        }
        cur_strs = strs;
        unsigned int* d_err = ctx->d_scratch->fp_flags;
        unsigned int* d_anynull = d_err + 1;
        TG_CUDA(ctx, cudaMemsetAsync(d_err, 0, 8, ctx->stream));
        const DProgram* dp = d_prog.as<DProgram>();
        int grid = tg_grid(ctx, n, FP_THREADS, 8);

        int64_t m = n;
        DevBuf sel;
        const int32_t* d_sel = nullptr;
        if (host_prog.filter_temp >= 0) {
            TG_TRY(jit_prepare(in));
            if (jit_project_chunks) {
                bool handled = false;
                TG_TRY(add_input_chunked(in, cols, strs, n, d_err, d_anynull, &handled, &m));
                if (handled) return TGPU_OK;
                // every row passed the filter: fall through to the identity form (blocks pass through, no copies)
            }
        }
        if (host_prog.filter_temp >= 0 && !jit_project_chunks) {
            DevBuf flags;
            TG_TRY(flags.alloc(ctx, (size_t)n));
            TG_TRY(jit_prepare(in));
            if (jit_filter) {
                long long n_arg = n;
                unsigned char* f_arg = flags.as<unsigned char>();
                void* params[5] = {&cols, &strs, &n_arg, &f_arg, &d_err};
                TG_TRY(jit_launch(ctx, jit_filter, tg_grid(ctx, n, FP_THREADS, jit_blocks_per_sm(jit_filter, FP_THREADS, 0)), FP_THREADS, 0, params));
            }
            else if (host_prog.has_dec) TG_LAUNCH(ctx, fp_filter_kernel<true>, grid, FP_THREADS, 0, dp, cols, strs, n, flags.as<uint8_t>(), d_err);
            else TG_LAUNCH(ctx, fp_filter_kernel<false>, grid, FP_THREADS, 0, dp, cols, strs, n, flags.as<uint8_t>(), d_err);
            long long* d_count = &ctx->d_scratch->fp_count;
            TG_TRY(tg_flagged_positions(ctx, flags.as<uint8_t>(), n, &sel, d_count));
            TG_TRY(tg_read_i64(ctx, d_count, &m));
            int64_t errw = 0;
            TG_TRY(tg_read_i64(ctx, d_err, &errw));
            TG_TRY(raise(errw));
            if (m == 0) return TGPU_OK;
            if (m < n) d_sel = sel.as<int32_t>();
        }

        DevPage outp;
        outp.rows = m;
        outp.cols.resize(projections.size());
        ComputedCols cc;
        for (size_t pi = 0; pi < projections.size(); pi++) {
            const tgpu_projection& pr = projections[pi];
            if (pr.kind == 0) {
                if (pr.index < 0 || pr.index >= (int32_t)in.cols.size()) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "projection channel out of range");
                if (!d_sel) outp.cols[pi] = in.cols[pr.index];       // InputPageProjection on all positions: the block itself
                else TG_TRY(tg_gather_column(ctx, in.cols[pr.index], d_sel, m, false, &outp.cols[pi]));
            }
            else TG_TRY(add_computed(pr, m, (int)pi, &outp, &cc));
        }
        if (cc.oc.count > 0 || cc.oc.str_count > 0) {
            int pgrid = tg_grid(ctx, m, FP_THREADS, 8);
            TG_TRY(jit_prepare(in));
            if (jit_project) {
                long long m_arg = m;
                void* params[7] = {&cols, &strs, &d_sel, &m_arg, &cc.oc, &d_err, &d_anynull};
                TG_TRY(jit_launch(ctx, jit_project, tg_grid(ctx, m, FP_THREADS, jit_blocks_per_sm(jit_project, FP_THREADS, 0)), FP_THREADS, 0, params));
            }
            else if (host_prog.has_dec) TG_LAUNCH(ctx, fp_project_kernel<true>, pgrid, FP_THREADS, 0, dp, cols, strs, d_sel, m, cc.oc, d_err, d_anynull);
            else TG_LAUNCH(ctx, fp_project_kernel<false>, pgrid, FP_THREADS, 0, dp, cols, strs, d_sel, m, cc.oc, d_err, d_anynull);
            TG_TRY(finish_computed(cc, d_err, &outp));
        }
        pending.push_back(tg_make_owned_page(std::move(outp)));
        return TGPU_OK;
    }

    // computed projection columns of one output page: their buffers as the project kernel sees them, and where they go
    struct ComputedCols {
        OutCols oc;
        std::vector<std::shared_ptr<DevBuf>> nullmaps;   // one byte per row, 1 = NULL
        std::vector<int> at;                             // output column of each computed column
        std::vector<std::shared_ptr<DevBuf>> str_bufs;   // VARCHAR projection k: descriptors 2k, null map 2k + 1
        std::vector<int> str_at;
        ComputedCols() { memset(&oc, 0, sizeof(oc)); }
    };

    // allocate output column `pi` (m rows) of computed projection `pr` and its byte null map
    int add_computed(const tgpu_projection& pr, int64_t m, int pi, DevPage* outp, ComputedCols* cc)
    {
        DevColumn& c = outp->cols[pi];
        if (pr.vtype == TGPU_V_VARCHAR) {
            // the piece descriptors and null map; finish_computed assembles the UTF8 column
            const int k = cc->oc.str_count++;
            c.type = TGPU_UTF8;
            c.length = m;
            auto desc = std::make_shared<DevBuf>(), nm = std::make_shared<DevBuf>();
            TG_TRY(desc->alloc(ctx, (size_t)m * host_prog.str_out[k].n * 8));
            TG_TRY(nm->alloc(ctx, (size_t)m));
            cc->oc.str_desc[k] = desc->p;
            cc->oc.str_nullmap[k] = nm->as<uint8_t>();
            cc->str_bufs.push_back(desc);
            cc->str_bufs.push_back(nm);
            cc->str_at.push_back(pi);
            return TGPU_OK;
        }
        const bool wide = pr.vtype == TGPU_V_DECIMAL && host_prog.temp_dec[pr.index] == 2;     // a long DECIMAL: 16-byte cells
        c.type = pr.vtype == TGPU_V_DOUBLE ? TGPU_FLOAT64 : pr.vtype == TGPU_V_BOOLEAN ? TGPU_INT8 : wide ? TGPU_INT128 : TGPU_INT64;
        c.length = m;
        c.own_data = std::make_shared<DevBuf>();
        TG_TRY(c.own_data->alloc(ctx, (size_t)m * c.elem_size()));
        c.data = c.own_data->p;
        auto nm = std::make_shared<DevBuf>();
        TG_TRY(nm->alloc(ctx, (size_t)m));
        int k = cc->oc.count++;
        cc->oc.temp[k] = pr.index;
        cc->oc.vtype[k] = wide ? TGD_V_DECIMAL_LONG : pr.vtype == TGPU_V_DECIMAL ? TGPU_V_BIGINT : pr.vtype;
        cc->oc.data[k] = c.own_data->p;
        cc->oc.nullmap[k] = nm->as<uint8_t>();
        cc->nullmaps.push_back(std::move(nm));
        cc->at.push_back(pi);
        return TGPU_OK;
    }

    // after the project kernel: raise its error bits, then give validity to the computed columns that hold a NULL
    int finish_computed(const ComputedCols& cc, unsigned int* d_err, DevPage* outp)
    {
        int64_t word = 0;
        TG_TRY(tg_read_i64(ctx, d_err, &word));
        TG_TRY(raise(word & 0xFFFFFFFFLL));
        uint32_t any_null = (uint32_t)((uint64_t)word >> 32);
        for (int k = 0; k < cc.oc.count; k++)
            if ((any_null >> k) & 1) TG_TRY(attach_validity(cc.nullmaps[k]->as<uint8_t>(), &outp->cols[cc.at[k]]));
        for (int k = 0; k < cc.oc.str_count; k++) TG_TRY(assemble_str(cc, k, d_err, &outp->cols[cc.str_at[k]]));
        return TGPU_OK;
    }

    // VARCHAR projection k: row lengths from the piece descriptors, a 64-bit scan to offsets (a column past utf8_limit bytes fails
    // before anything is written), then the bytes
    int assemble_str(const ComputedCols& cc, int k, unsigned int* d_any, DevColumn* c)
    {
        const DStrOut& so = host_prog.str_out[k];
        const int64_t m = c->length;
        const int2* desc = (const int2*)cc.oc.str_desc[k];
        const uint8_t* nullmap = cc.oc.str_nullmap[k];
        DevBuf len, off64;
        TG_TRY(len.alloc(ctx, (size_t)(m + 1) * 8));
        TG_TRY(off64.alloc(ctx, (size_t)(m + 1) * 8));
        TG_CUDA(ctx, cudaMemsetAsync(d_any, 0, 4, ctx->stream));
        TG_LAUNCH(ctx, fp_str_lengths_kernel, tg_grid(ctx, m, 256, 8), 256, 0, desc, so.n, nullmap, m, len.as<long long>(), d_any);
        TG_TRY(tg_exclusive_sum(ctx, len.as<long long>(), off64.as<long long>(), m + 1));
        int64_t total = 0, any = 0;
        TG_TRY(tg_read_i64(ctx, off64.as<long long>() + m, &total));
        TG_TRY(tg_read_i64(ctx, d_any, &any));
        if (total > utf8_limit)
            return tg_fail(ctx, TGPU_ERR_INSUFFICIENT_RESOURCES, "VARCHAR projection %d holds %lld bytes, past the %lld a UTF8 column holds", k, (long long)total,
                           (long long)utf8_limit);
        c->own_offsets = std::make_shared<DevBuf>();
        TG_TRY(c->own_offsets->alloc(ctx, (size_t)(m + 1) * 4));
        TG_LAUNCH(ctx, fp_str_narrow_kernel, tg_grid(ctx, m + 1, 256, 8), 256, 0, off64.as<long long>(), m + 1, c->own_offsets->as<int32_t>());
        c->offsets = c->own_offsets->as<int32_t>();
        c->own_data = std::make_shared<DevBuf>();
        TG_TRY(c->own_data->alloc(ctx, (size_t)total));
        c->data = c->own_data->p;
        c->data_bytes = total;
        StrSrcs srcs;
        memset(&srcs, 0, sizeof(srcs));
        for (int q = 0; q < so.n; q++) {
            const int32_t src = so.src[q];
            if (src == TGD_SRC_NONE) srcs.base[q] = nullptr;
            else if (src >= 0) srcs.base[q] = cur_strs.bytes[host_prog.str_slot[src]];
            else srcs.base[q] = d_prog.as<uint8_t>() + offsetof(DProgram, str_bytes) + host_prog.str_off[-(src + 1)];
        }
        if (total > 0) {
            const int64_t tiles = tg_div_up(m, 32);
            TG_LAUNCH(ctx, fp_str_assemble_kernel, tg_grid(ctx, tiles, FPS_WARPS, 8), FPS_WARPS * 32, 0, desc, so.n, srcs, c->offsets, m,
                      c->own_data->as<uint8_t>());
        }
        if (any & 0xFFFFFFFFLL) TG_TRY(attach_validity(nullmap, c));
        return TGPU_OK;
    }

    // pack the byte null map of c's rows into its validity bitmap
    int attach_validity(const uint8_t* nullmap, DevColumn* c)
    {
        c->own_validity = std::make_shared<DevBuf>();
        TG_TRY(c->own_validity->alloc(ctx, (size_t)((c->length + 7) / 8)));
        TG_TRY(tg_pack_nullmap(ctx, nullmap, c->length, c->own_validity->as<uint8_t>()));
        c->validity = c->own_validity->as<uint8_t>();
        return TGPU_OK;
    }

    // chunked two-pass form: handled = false (and *m_out = n) when every row is selected
    int add_input_chunked(const DevPage& in, const DColumns& cols, const StrCols& strs_in, int64_t n, unsigned int* d_err, unsigned int* d_anynull, bool* handled,
                          int64_t* m_out)
    {
        *handled = false;
        const int64_t tile = (int64_t)FPC_R * FPC_T;
        int per_sm = std::min(jit_blocks_per_sm(jit_filter_chunks, FPC_T, 0), jit_blocks_per_sm(jit_project_chunks, FPC_T, 0));
        int64_t want = std::min<int64_t>(tg_div_up(n, tile), (int64_t)ctx->sm_count * per_sm);
        long long chunk = (long long)(tg_div_up(tg_div_up(n, want), tile) * tile);
        int chunks = (int)tg_div_up(n, chunk);
        DevBuf flags, counts, chunk_off, d_total;
        TG_TRY(flags.alloc(ctx, (size_t)n));
        TG_TRY(counts.alloc(ctx, (size_t)chunks * 4));
        TG_TRY(chunk_off.alloc(ctx, (size_t)chunks * 8));
        TG_TRY(d_total.alloc(ctx, 8));
        long long n_arg = n;
        {
            DColumns c = cols;
            StrCols sc = strs_in;
            unsigned char* f_arg = flags.as<unsigned char>();
            unsigned int* cnt_arg = counts.as<unsigned int>();
            void* params[7] = {&c, &sc, &n_arg, &chunk, &f_arg, &cnt_arg, &d_err};
            TG_TRY(jit_launch(ctx, jit_filter_chunks, chunks, FPC_T, 0, params));
        }
        TG_LAUNCH(ctx, fp_chunk_scan_kernel, 1, 256, 0, counts.as<unsigned int>(), chunks, chunk_off.as<long long>(), d_total.as<long long>());
        int64_t m = 0, errw = 0;
        TG_TRY(tg_read_i64(ctx, d_total.p, &m));
        TG_TRY(tg_read_i64(ctx, d_err, &errw));
        TG_TRY(raise(errw & 0xFFFFFFFFLL));
        *m_out = m;
        if (m == n) return TGPU_OK;
        *handled = true;
        if (m == 0) return TGPU_OK;
        DevPage outp;
        outp.rows = m;
        outp.cols.resize(projections.size());
        ComputedCols cc;
        OutCols& oc = cc.oc;
        std::vector<std::shared_ptr<DevBuf>> pass_nullmaps;
        std::vector<int> pass_at;
        for (size_t pi = 0; pi < projections.size(); pi++) {
            const tgpu_projection& pr = projections[pi];
            if (pr.kind == 0) {
                if (pr.index < 0 || pr.index >= (int32_t)in.cols.size()) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "projection channel out of range");
                const DevColumn& src = in.cols[pr.index];
                DevColumn& c = outp.cols[pi];
                c.type = src.type;
                c.length = m;
                c.own_data = std::make_shared<DevBuf>();
                TG_TRY(c.own_data->alloc(ctx, (size_t)m * src.elem_size()));
                c.data = c.own_data->p;
                int k = oc.pass_count++;
                oc.pass_data[k] = c.own_data->p;
                std::shared_ptr<DevBuf> nm;
                if (src.validity) {
                    nm = std::make_shared<DevBuf>();
                    TG_TRY(nm->alloc(ctx, (size_t)m));
                    oc.pass_nullmap[k] = nm->as<uint8_t>();
                }
                pass_nullmaps.push_back(nm);
                pass_at.push_back((int)pi);
            }
            else TG_TRY(add_computed(pr, m, (int)pi, &outp, &cc));
        }
        {
            DColumns c = cols;
            StrCols sc = strs_in;
            const unsigned char* f_arg = flags.as<unsigned char>();
            const long long* off_arg = chunk_off.as<long long>();
            void* params[9] = {&c, &sc, &f_arg, &n_arg, &chunk, &off_arg, &oc, &d_err, &d_anynull};
            TG_TRY(jit_launch(ctx, jit_project_chunks, chunks, FPC_T, 0, params));
        }
        TG_TRY(finish_computed(cc, d_err, &outp));
        for (int k = 0; k < oc.pass_count; k++)
            if (pass_nullmaps[k]) TG_TRY(attach_validity(pass_nullmaps[k]->as<uint8_t>(), &outp.cols[pass_at[k]]));
        pending.push_back(tg_make_owned_page(std::move(outp)));
        return TGPU_OK;
    }

    // kernels specialised for this program and this page's channel types / nullability (NVRTC, cached)
    void* jit_filter = nullptr;
    void* jit_project = nullptr;
    void* jit_filter_chunks = nullptr;      // chunked two-pass form (nullptr: not applicable to this program / page shape)
    void* jit_project_chunks = nullptr;
    std::string jit_key;
    std::vector<int> pass_channels() const
    {
        std::vector<int> v;
        for (auto& pr : projections)
            if (pr.kind == 0) v.push_back(pr.index);
        return v;
    }
    int jit_prepare(const DevPage& in)
    {
        if (!jit_available()) { jit_filter = jit_project = nullptr; return TGPU_OK; }
        int elems[TGPU_MAX_CHANNELS] = {0};
        uint32_t nullable = 0;
        std::string key;
        for (size_t c = 0; c < in.cols.size() && c < TGPU_MAX_CHANNELS; c++) {
            elems[c] = in.cols[c].elem_size();
            if (in.cols[c].validity) nullable |= 1u << c;
            key += (char)('0' + elems[c]);
        }
        key += ":" + std::to_string(nullable);
        if (key == jit_key && jit_filter) return TGPU_OK;
        std::vector<int> pass = pass_channels();
        std::string src = gen_fp_source(host_prog, elems, (int)in.cols.size(), nullable, pass);
        TG_TRY(jit_get_function(ctx, src, "tg_fp_filter_jit", &jit_filter));
        TG_TRY(jit_get_function(ctx, src, "tg_fp_project_jit", &jit_project));
        jit_filter_chunks = jit_project_chunks = nullptr;
        if (src.find("tg_fp_project_chunks_jit") != std::string::npos && pass.size() <= TGPU_MAX_CHANNELS && !getenv("TGPU_FP_SELECTION_VECTOR")) {
            TG_TRY(jit_get_function(ctx, src, "tg_fp_filter_chunks_jit", &jit_filter_chunks));
            TG_TRY(jit_get_function(ctx, src, "tg_fp_project_chunks_jit", &jit_project_chunks));
        }
        jit_key = key;
        return TGPU_OK;
    }

    int raise(int64_t errbits)
    {
        // in a program with DECIMAL the invalid-cast bit may come from a DECIMAL cast as well as from CAST(DOUBLE AS BIGINT)
        if (host_prog.has_dec && !(errbits & (TG_ERR_BIT_DIV_ZERO | TG_ERR_BIT_OVERFLOW)) && (errbits & TG_ERR_BIT_INVALID_CAST))
            return tg_fail(ctx, TGPU_ERR_INVALID_CAST_ARGUMENT, "Cannot cast value: it does not fit the target type");
        return expr_raise(ctx, errbits);
    }

    int get_output(OwnedPage** out) override
    {
        *out = nullptr;
        if (next_out < pending.size()) *out = pending[next_out++];
        return TGPU_OK;
    }
    int finish() override { finishing = true; return TGPU_OK; }
    bool is_finished() override { return finishing && next_out >= pending.size(); }
};

}  // namespace

extern "C" int tgpu_filter_project_create(tgpu_ctx* ctx, const tgpu_expr_program* program, tgpu_op** out)
{
    if (!ctx || !program || !out) return TGPU_ERR_INVALID_ARGUMENT;
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    std::unique_ptr<FilterProjectOp> op(new FilterProjectOp(ctx));
    TG_TRY(tg::expr_compile(ctx, program, &op->host_prog, &op->max_channel));
    // a smaller byte limit for VARCHAR projection columns, so that the INT32_MAX guard can be exercised on small pages
    if (const char* lim = getenv("TGPU_UTF8_COLUMN_LIMIT")) op->utf8_limit = std::min<int64_t>(INT32_MAX, std::max<int64_t>(0, atoll(lim)));
    if (program->num_projections > TGPU_MAX_CHANNELS) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "more than %d projections", TGPU_MAX_CHANNELS);
    for (int i = 0; i < program->num_projections; i++) {
        const tgpu_projection& p = program->projections[i];
        if (p.kind == 1 && (p.index < 0 || p.index >= TGPU_MAX_TEMPS)) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "projection temp out of range");
        if (p.kind == 1 && p.vtype == TGPU_V_DECIMAL && op->host_prog.temp_dec[p.index] == 0)
            return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "projection %d: temp %d does not hold a DECIMAL", i, p.index);
        if (p.kind == 1 && p.vtype != TGPU_V_DECIMAL && op->host_prog.temp_dec[p.index] != 0)
            return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "projection %d: temp %d holds a DECIMAL, the projection's type is %d", i, p.index, p.vtype);
        op->projections.push_back(p);
    }
    TG_TRY(op->d_prog.alloc(ctx, sizeof(tg::DProgram)));
    TG_CUDA(ctx, cudaMemcpyAsync(op->d_prog.p, &op->host_prog, sizeof(tg::DProgram), cudaMemcpyHostToDevice, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    *out = op.release();
    return TGPU_OK;
}

extern "C" int tgpu_jit_selftest_filter_project(const tgpu_expr_program* program, const int32_t* channel_types, int32_t num_channels, uint32_t nullable_mask,
                                                int64_t* cubin_bytes, char* source_out, int64_t source_cap)
{
    if (!program || !channel_types || !cubin_bytes) return TGPU_ERR_INVALID_ARGUMENT;
    tgpu_ctx fake;
    tg::DProgram prog;
    int32_t max_channel = -1;
    int st = tg::expr_compile(&fake, program, &prog, &max_channel);
    if (st != TGPU_OK) return st;
    std::vector<int> pass;
    for (int32_t i = 0; i < program->num_projections; i++)
        if (program->projections[i].kind == 0) pass.push_back(program->projections[i].index);
    return tg::jit_selftest(channel_types, num_channels, [&](const int* elems) {
        return gen_fp_source(prog, elems, num_channels, nullable_mask, pass);
    }, cubin_bytes, source_out, source_cap);
}
