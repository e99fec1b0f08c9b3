// Test and benchmark hooks of the kernels (C ABI wl_test_* / wl_bench_gemm): each runs one kernel, or the code the
// engine runs around it, on its own device copies of the caller's inputs.
#include <cstring>

#include "ctx.cuh"

static __half* upload_fill_f16(Scratch& sc, size_t n, float v) {
  std::vector<__half> h(n, __float2half_rn(v));
  return sc.upload(h.data(), n);
}
static void download_f16(Scratch& sc, const __half* d, float* out, size_t n) {
  std::vector<__half> h(n);
  sc.download(h.data(), d, n);
  for (size_t i = 0; i < n; ++i) out[i] = __half2float(h[i]);
}

extern "C" int wl_test_gemm(wl_ctx* c, const uint16_t* a_f16, const uint16_t* b_f16, const float* bias, float* cc, int32_t M,
                            int32_t N, int32_t K, int32_t batch, int32_t transposed_store, int32_t gelu, int32_t use_simt,
                            int32_t opts) {
  API_BEGIN(c)
  const int out_kind = opts & 3, variant = (opts >> 4) & 3, hs_S = opts >> 8;
  const bool a_shared = opts & 4, b_shared = opts & 8, bias_on_m = transposed_store || (opts & 64);
  const bool f16_out = out_kind == 2 || out_kind == 3;
  WL_CHECK(variant <= GEMM_PINGPONG && (out_kind != 3 || (hs_S > 0 && M % hs_S == 0 && N % 64 == 0 && batch == 1)), WL_ERR_ARG,
           "wl_test_gemm: bad opts %d", opts);
  const size_t na = (size_t)(a_shared ? 1 : batch) * M * K, nb = (size_t)(b_shared ? 1 : batch) * N * K, nc = (size_t)batch * M * N;
  Scratch sc(c->st);
  const __half* da = sc.upload(reinterpret_cast<const __half*>(a_f16), na);
  const __half* db = sc.upload(reinterpret_cast<const __half*>(b_f16), nb);
  float* dc = out_kind == 1 ? sc.upload(cc, nc) : sc.alloc<float>(nc, 0);   // out_kind 1: the residual, updated in place
  __half* dh = sc.alloc<__half>(nc, 0);
  float* dbias = nullptr;
  if (bias) {
    dbias = sc.alloc<float>((size_t)std::max(M, N));
    WL_CUDA(cudaMemcpyAsync(dbias, bias, (size_t)(bias_on_m ? M : N) * 4, cudaMemcpyHostToDevice, c->st));
  }
  int* dslots = nullptr;
  if (out_kind == 3) {   // head-split into slots in reverse stream order: out[slot][h][s][64], s-swizzled 16-byte pieces
    const int ns = M / hs_S;
    std::vector<int> slots(ns);
    for (int b = 0; b < ns; ++b) slots[b] = ns - 1 - b;
    dslots = sc.upload(slots.data(), ns);
  }
  GemmEpilogue e;
  e.out = f16_out ? (void*)dh : (void*)dc; e.out_f32 = f16_out ? 0 : 1; e.gelu = gelu; e.bias = dbias;
  if (transposed_store) { e.ldm = 1; e.ldn = M; }   // C^T stored: [N][M]
  else { e.ldm = N; e.ldn = 1; }
  e.bias_on_m = bias_on_m;
  e.ob1 = (long)M * N;
  if (out_kind == 1) { e.resid = dc; e.rldm = e.ldm; e.rldn = e.ldn; e.rb1 = e.ob1; }
  if (out_kind == 3) {
    e.mode = GEMM_HEADSPLIT; e.hs_S = hs_S; e.hs_H = N / 64; e.hs_slot_stride = (long)hs_S * N; e.hs_slots = dslots;
  }
  GemmOperand A = opnd(da, M, K, K, batch, a_shared ? 0 : (long)M * K), Bo = opnd(db, N, K, K, batch, b_shared ? 0 : (long)N * K);
  if (a_shared) A.n1 = 1;
  if (b_shared) Bo.n1 = 1;
  if (use_simt) gemm_tn_simt(c->st, A, Bo, M, N, K, e);
  else gemm_tn(c->st, A, Bo, M, N, K, e, (GemmVariant)variant);
  if (f16_out) download_f16(sc, dh, cc, nc);
  else sc.download(cc, dc, nc);
  API_END(c)
}

extern "C" int wl_gemm_variant(wl_ctx* c, int32_t M, int32_t N, int32_t K, int32_t batch, int32_t* variant_out) {
  API_BEGIN(c)
  WL_CHECK(variant_out && M > 0 && N > 0 && K > 0 && batch > 0, WL_ERR_ARG, "wl_gemm_variant: bad arguments");
  *variant_out = (int32_t)gemm_tn_variant(M, N, K, batch);
  API_END(c)
}

// mode 0/1/2/3 of wgemm (see gemm.cuh); out holds [R][n_out] floats (mode 1: the residual on input, the sum on output;
// mode 2: gelu as fp32; mode 3: the K ranges summed on the host side of this hook)
extern "C" int wl_test_wgemm(wl_ctx* c, const uint16_t* w_f16, const uint16_t* x_f16, const float* bias, float* out, int32_t R,
                             int32_t n_out, int32_t K, int32_t mode) {
  API_BEGIN(c)
  WL_CHECK(w_f16 && x_f16 && out && mode >= 0 && mode <= 3, WL_ERR_ARG, "wl_test_wgemm: bad arguments");
  WL_CHECK(wgemm_supported(R, K), WL_ERR_ARG, "wl_test_wgemm: unsupported shape R=%d K=%d", R, K);
  const size_t nw = (size_t)n_out * K, nx = (size_t)R * K, no = (size_t)R * n_out;
  const int ks = wgemm_ksplit(K);
  Scratch sc(c->st);
  const __half* dw = sc.upload(reinterpret_cast<const __half*>(w_f16), nw);
  const __half* dx = sc.upload(reinterpret_cast<const __half*>(x_f16), nx);
  __half* dh = sc.alloc<__half>(no);
  float* dout = sc.alloc<float>(no * (size_t)std::max(1, ks), 0);
  if (mode == 1) WL_CUDA(cudaMemcpyAsync(dout, out, no * 4, cudaMemcpyHostToDevice, c->st));
  const float* db = bias ? sc.upload(bias, n_out) : nullptr;
  wgemm(c->st, dw, n_out, K, dx, R, db, mode, dout, dh, (long)no);
  if (mode == 2) {
    download_f16(sc, dh, out, no);
  } else if (mode == 3) {
    std::vector<float> h(no * ks);
    sc.download(h.data(), dout, h.size());
    for (size_t i = 0; i < no; ++i) { float a = 0.f; for (int q = 0; q < ks; ++q) a += h[(size_t)q * no + i]; out[i] = a; }
  } else {
    sc.download(out, dout, no);
  }
  API_END(c)
}

extern "C" int wl_test_dec_gemm(wl_ctx* c, const uint16_t* w_f16, const uint16_t* x_f16, float* out, int32_t R, int32_t n_out,
                                int32_t K, int32_t nsplit, int32_t* nsplit_out) {
  API_BEGIN(c)
  PdlScope pdl(false);
  WL_CHECK(w_f16 && x_f16 && nsplit_out && R > 0 && n_out > 0 && K > 0 && K % 8 == 0 && nsplit >= 0, WL_ERR_ARG,
           "wl_test_dec_gemm: bad arguments");
  const int ns = nsplit == 0 ? dec_gemm_split_plan(n_out, R, K, 8) : nsplit;
  const int kb = cdiv(K, 64);
  WL_CHECK(cdiv(kb, cdiv(kb, ns)) == ns, WL_ERR_ARG, "wl_test_dec_gemm: %d K ranges cannot be formed from %d k-blocks", ns, kb);
  *nsplit_out = ns;
  if (!out) return WL_OK;   // split query only
  Scratch sc(c->st);
  const long part = (long)R * n_out;
  const __half* dw = sc.upload(reinterpret_cast<const __half*>(w_f16), (size_t)n_out * K);
  const __half* dx = sc.upload(reinterpret_cast<const __half*>(x_f16), (size_t)R * K);
  float* dout = sc.alloc<float>((size_t)ns * part, 0xff);   // NaN: an element no K range wrote cannot pass as a value
  dec_gemm(c->st, dw, n_out, K, dx, R, dout, n_out, part, ns);
  sc.download(out, dout, (size_t)ns * part);
  API_END(c)
}

extern "C" int wl_test_cross_attn(wl_ctx* c, const float* q_part, const float* q_bias, int32_t q_nsplit, const uint16_t* k_pool,
                                  const uint16_t* v_pool, int32_t n_slots, const int32_t* slot, const int32_t* done, int32_t B,
                                  int32_t rows_per_stream, int32_t H, int32_t nsplit, int32_t* nsplit_out, float sentinel,
                                  float* out, float* probs) {
  API_BEGIN(c)
  PdlScope pdl(false);
  WL_CHECK(q_part && k_pool && v_pool && slot && done && out && nsplit_out && B > 0 && H > 0 && n_slots > 0 && nsplit >= 0 &&
               rows_per_stream >= 1 && rows_per_stream <= MAX_ROWS_PER_STREAM,
           WL_ERR_ARG, "wl_test_cross_attn: bad arguments");
  for (int b = 0; b < B; ++b) WL_CHECK(slot[b] >= 0 && slot[b] < n_slots, WL_ERR_ARG, "wl_test_cross_attn: slot %d out of range", slot[b]);
  const int nchunk = cdiv(S_ENC, 128);
  const int ns = nsplit == 0 ? cross_attn_pick_nsplit(B, H, c->num_sms, rows_per_stream) : nsplit;
  WL_CHECK(ns >= 1 && ns <= nchunk && cdiv(nchunk, cdiv(nchunk, ns)) == ns, WL_ERR_ARG,
           "wl_test_cross_attn: %d key ranges cannot be formed from %d chunks", ns, nchunk);
  WL_CHECK(!probs || ns == 1, WL_ERR_ARG, "wl_test_cross_attn: the probabilities need the whole key range (nsplit 1)");
  *nsplit_out = ns;
  const int d = H * 64, R = B * rows_per_stream;
  const long slot_sz = (long)S_ENC * d;
  Scratch sc(c->st);
  DecodeState s;
  memset(&s, 0, sizeof(s));   // the two kernels read only slot and done
  s.slot = sc.upload(slot, B);
  s.done = sc.upload(done, B);
  PartialSrc q;
  q.nsplit = q_nsplit;
  q.stride = (long)R * d;
  q.ptr = sc.upload(q_part, (size_t)std::max(q_nsplit, 1) * R * d);
  q.bias = q_bias ? sc.upload(q_bias, d) : nullptr;
  const __half* kc = sc.upload(reinterpret_cast<const __half*>(k_pool), (size_t)n_slots * slot_sz);
  const __half* vc = sc.upload(reinterpret_cast<const __half*>(v_pool), (size_t)n_slots * slot_sz);
  CrossAttnWorkspace ws;
  ws.part = sc.alloc<float>((size_t)B * H * ns * MAX_ROWS_PER_STREAM * 66);
  ws.probs = probs ? sc.alloc<float>((size_t)R * H * S_ENC, 0) : nullptr;
  __half* dout = upload_fill_f16(sc, (size_t)R * d, sentinel);
  decoder_cross_attn(c->st, s, q, kc, vc, slot_sz, ws, dout, B, rows_per_stream, H, d, ns);
  download_f16(sc, dout, out, (size_t)R * d);
  if (probs) sc.download(probs, ws.probs, (size_t)R * H * S_ENC);
  API_END(c)
}

extern "C" int wl_test_self_attn(wl_ctx* c, const float* qkv_part, const float* qkv_bias, int32_t nsplit, uint16_t* k_cache,
                                 uint16_t* v_cache, int32_t n_rows, const int16_t* src, const int32_t* pos, const int32_t* active,
                                 const int32_t* wrow, int32_t R, int32_t H, float sentinel, float* out) {
  API_BEGIN(c)
  PdlScope pdl(false);
  WL_CHECK(qkv_part && k_cache && v_cache && src && pos && active && out && R > 0 && H > 0 && n_rows > 0 && nsplit >= 1 &&
               nsplit <= 8,
           WL_ERR_ARG, "wl_test_self_attn: bad arguments");
  for (int r = 0; r < R; ++r) {
    WL_CHECK(pos[r] >= 0 && pos[r] < T_MAX && (wrow ? wrow[r] : r) >= 0 && (wrow ? wrow[r] : r) < n_rows, WL_ERR_ARG,
             "wl_test_self_attn: row %d: position or write row out of range", r);
    for (int p = 0; active[r] && p < pos[r]; ++p)
      WL_CHECK(src[(long)r * T_MAX + p] >= 0 && src[(long)r * T_MAX + p] < n_rows, WL_ERR_ARG, "wl_test_self_attn: src out of range");
  }
  const int d = H * 64;
  const long row_stride = (long)H * T_MAX * 64;
  Scratch sc(c->st);
  DecodeState s;
  memset(&s, 0, sizeof(s));   // the kernel reads only src, pos, active and wrow
  s.src = sc.upload(src, (size_t)R * T_MAX);
  s.pos = sc.upload(pos, R);
  s.active = sc.upload(active, R);
  s.wrow = wrow ? sc.upload(wrow, R) : nullptr;
  PartialSrc qkv;
  qkv.nsplit = nsplit;
  qkv.stride = (long)R * 3 * d;
  qkv.ptr = sc.upload(qkv_part, (size_t)nsplit * R * 3 * d);
  qkv.bias = qkv_bias ? sc.upload(qkv_bias, 3 * d) : nullptr;
  __half* kc = sc.upload(reinterpret_cast<__half*>(k_cache), (size_t)n_rows * row_stride);
  __half* vc = sc.upload(reinterpret_cast<__half*>(v_cache), (size_t)n_rows * row_stride);
  __half* dout = upload_fill_f16(sc, (size_t)R * d, sentinel);
  decoder_self_attn(c->st, s, qkv, kc, vc, row_stride, dout, R, H, d);
  download_f16(sc, dout, out, (size_t)R * d);
  sc.download(reinterpret_cast<__half*>(k_cache), kc, (size_t)n_rows * row_stride);
  sc.download(reinterpret_cast<__half*>(v_cache), vc, (size_t)n_rows * row_stride);
  API_END(c)
}

extern "C" int wl_test_fold(wl_ctx* c, int32_t mode, float* x, const float* part, int32_t nsplit, const float* bias,
                            const float* gamma, const float* beta, float* y, int32_t rows, int32_t cols) {
  API_BEGIN(c)
  PdlScope pdl(false);
  WL_CHECK(y && rows > 0 && cols > 0 && (mode == 0 || mode == 1) && nsplit >= 0 && nsplit <= 8 && (nsplit == 0 || part),
           WL_ERR_ARG, "wl_test_fold: bad arguments");
  WL_CHECK(mode == 1 || (x && gamma && beta), WL_ERR_ARG, "wl_test_fold: layernorm_update needs x, gamma and beta");
  WL_CHECK(mode == 0 || nsplit >= 1, WL_ERR_ARG, "wl_test_fold: gelu_cast needs at least one K range");
  const size_t n = (size_t)rows * cols;
  Scratch sc(c->st);
  PartialSrc upd;
  upd.nsplit = nsplit;
  upd.stride = (long)n;
  upd.ptr = nsplit ? sc.upload(part, (size_t)nsplit * n) : nullptr;
  upd.bias = bias ? sc.upload(bias, cols) : nullptr;
  __half* dy = sc.alloc<__half>(n, 0);
  float* dx = mode == 0 ? sc.upload(x, n) : nullptr;
  const float* dg = mode == 0 ? sc.upload(gamma, cols) : nullptr;
  const float* db = mode == 0 ? sc.upload(beta, cols) : nullptr;
  if (mode == 0) layernorm_update_rows(c->st, dx, upd, dg, db, dy, rows, cols);
  else gelu_cast(c->st, upd, dy, rows, cols);
  download_f16(sc, dy, y, n);
  if (mode == 0) sc.download(x, dx, n);
  API_END(c)
}

// Test hooks of the encoder-pass kernels: each runs the code encoder_pass runs, on its own device copies of the inputs.
extern "C" int wl_test_enc_attn(wl_ctx* c, const uint16_t* qk_f16, const uint16_t* vt_f16, uint16_t* out_f16, int32_t nb,
                                int32_t H, int32_t path, int32_t ab) {
  API_BEGIN(c)
  WL_CHECK(qk_f16 && vt_f16 && out_f16 && nb >= 1 && H >= 1 && H <= 32 && (path == 0 || path == 1) && ab >= 0, WL_ERR_ARG,
           "wl_test_enc_attn: bad arguments");
  const int d = H * 64;
  const size_t n_qk = (size_t)nb * S_ENC * 2 * d, n_vt = (size_t)nb * d * S_PAD, n_out = ((size_t)nb * S_ENC + 128) * d;
  Scratch sc(c->st);
  const __half* dqk = sc.upload(reinterpret_cast<const __half*>(qk_f16), n_qk);
  const __half* dvt = sc.upload(reinterpret_cast<const __half*>(vt_f16), n_vt);
  __half* dout = sc.upload(reinterpret_cast<const __half*>(out_f16), n_out);
  if (path == 0) {
    encoder_attention_fused(c->st, dqk, dvt, dout, nb, H, d);
  } else {
    const int AB = ab ? ab : std::min(nb, enc_attn_streams(d));
    // zeroed like the engine's workspaces: the scores GEMM never writes the pad columns, softmax_rows writes all of P
    float* scores = sc.alloc<float>((size_t)AB * H * S_ENC * S_PAD, 0);
    __half* probs16 = sc.alloc<__half>((size_t)AB * H * S_ENC * S_PAD, 0);
    encoder_attention_unfused(c->st, dqk, dvt, dout, scores, probs16, nb, H, AB);
  }
  sc.download(reinterpret_cast<__half*>(out_f16), dout, n_out);
  API_END(c)
}

extern "C" int wl_test_enc_stem(wl_ctx* c, const float* feats_f32, float* x_out_f32, int32_t nb) {
  API_BEGIN(c)
  WL_CHECK(c->finalized, WL_ERR_STATE, "weights not finalized");
  WL_CHECK(feats_f32 && x_out_f32 && nb >= 1, WL_ERR_ARG, "wl_test_enc_stem: bad arguments");
  const int d = c->d, nm = c->n_mels;
  Scratch sc(c->st);
  const float* dfeat = sc.upload(feats_f32, (size_t)nb * nm * 3000);
  // the engine's shapes, slack included; zeroed: rows 0 and 3001 of every stream are the conv padding
  const size_t n16 = (size_t)nb * 3002 * nm + 4096, n1 = (size_t)nb * 3002 * d + 4096, nx = (size_t)nb * S_ENC * d;
  __half* feat16 = sc.alloc<__half>(n16, 0);
  __half* conv1o = sc.alloc<__half>(n1, 0);
  float* x = sc.alloc<float>(nx, 0xff);   // NaN: an element the stem did not write cannot pass as a value
  encoder_stem(c, c->st, nb, dfeat, feat16, conv1o, x);
  sc.download(x_out_f32, x, nx);
  API_END(c)
}

extern "C" int wl_test_layernorm(wl_ctx* c, const float* x_f32, const float* gamma, const float* beta, float* y16_as_f32,
                                 float* y32, int32_t rows, int32_t d) {
  API_BEGIN(c)
  WL_CHECK(x_f32 && gamma && beta && rows >= 1 && d >= 4, WL_ERR_ARG, "wl_test_layernorm: bad arguments");
  // the outputs carry 8 guard rows after the last one: the grid covers whole blocks of 8 rows
  const size_t n = (size_t)rows * d, ng = (size_t)(rows + 8) * d;
  Scratch sc(c->st);
  const float* dx = sc.upload(x_f32, n);
  const float* dg = sc.upload(gamma, d);
  const float* db = sc.upload(beta, d);
  __half* dy = nullptr;
  float* dy32 = nullptr;
  if (y16_as_f32) {
    std::vector<__half> h(ng);
    for (size_t i = 0; i < ng; ++i) h[i] = __float2half_rn(y16_as_f32[i]);
    dy = sc.upload(h.data(), ng);
  }
  if (y32) dy32 = sc.upload(y32, ng);
  layernorm_rows(c->st, dx, dg, db, dy, dy32, rows, d);
  if (y16_as_f32) download_f16(sc, dy, y16_as_f32, ng);
  if (y32) sc.download(y32, dy32, ng);
  API_END(c)
}

// A tensor wl_load_tensor / wl_load_tensor_typed uploaded, as the device holds it (fp32 or fp16 bytes, after the conv
// re-layout), before wl_finalize_weights.
extern "C" int wl_test_read_weight(wl_ctx* c, const char* name, void* out) {
  API_BEGIN(c)
  WL_CHECK(name && out, WL_ERR_ARG, "wl_test_read_weight: bad arguments");
  const std::string nm(name);
  auto it = c->dev.find(nm);
  WL_CHECK(it != c->dev.end(), WL_ERR_ARG, "wl_test_read_weight: no weight '%s'", name);
  const auto& sh = c->shape[nm];
  size_t n = 1;
  for (auto s : sh) n *= (size_t)s;
  const bool as_f32 = sh.size() == 1 || nm == "model.encoder.embed_positions.weight" || nm == "mel_filters";
  WL_CUDA(cudaStreamSynchronize(c->st));
  WL_CUDA(cudaMemcpy(out, it->second, n * (as_f32 ? sizeof(float) : sizeof(__half)), cudaMemcpyDeviceToHost));
  API_END(c)
}

extern "C" int wl_bench_gemm(wl_ctx* c, int32_t M, int32_t N, int32_t K, int32_t batch, int32_t iters, int32_t flags,
                             float* ms_out) {
  // flags: 1 transposed (swap-AB) store, 2 bias, 4 GELU, 8 fp32 output with fp32 residual (in place), 16 bias on m,
  // 32 A shared by the batch, 64 output rows padded to a multiple of 64 elements (V^T: S_PAD)
  API_BEGIN(c)
  WL_CHECK(ms_out && M > 0 && N > 0 && K > 0 && batch > 0 && iters > 0, WL_ERR_ARG, "wl_bench_gemm: bad arguments");
  const bool tr = flags & 1, f32 = flags & 8, a_shared = flags & 32;
  const long ld = (flags & 64) ? (N + 63) / 64 * 64 : N;
  const size_t na = (size_t)(a_shared ? 1 : batch) * M * K, nb = (size_t)batch * N * K, nc = (size_t)batch * M * ld;
  Scratch sc(c->st);
  const __half* da = sc.alloc<__half>(na, 0x11);
  const __half* db = sc.alloc<__half>(nb, 0x11);
  void* dc = f32 ? (void*)sc.alloc<float>(nc, 0) : (void*)sc.alloc<__half>(nc, 0);
  const float* dbias = sc.alloc<float>((size_t)std::max(M, N), 0);
  GemmEpilogue e;
  e.out = dc; e.out_f32 = f32 ? 1 : 0;
  if (tr) { e.ldm = 1; e.ldn = M; } else { e.ldm = ld; e.ldn = 1; }
  e.ob1 = (long)M * ld;
  if (flags & 2) { e.bias = dbias; e.bias_on_m = (tr || (flags & 16)) ? 1 : 0; }
  if (flags & 4) e.gelu = 1;
  if (f32) { e.resid = (const float*)dc; e.rldm = e.ldm; e.rldn = e.ldn; e.rb1 = e.ob1; }
  GemmOperand A = opnd(da, M, K, K, a_shared ? 1 : batch, a_shared ? 0 : (long)M * K), Bo = opnd(db, N, K, K, batch, (long)N * K);
  for (int i = 0; i < 3; ++i) gemm_tn(c->st, A, Bo, M, N, K, e);
  WL_CUDA(cudaEventRecord(c->ev0, c->st));
  for (int i = 0; i < iters; ++i) gemm_tn(c->st, A, Bo, M, N, K, e);
  WL_CUDA(cudaEventRecord(c->ev1, c->st));
  WL_CUDA(cudaStreamSynchronize(c->st));
  float ms;
  WL_CUDA(cudaEventElapsedTime(&ms, c->ev0, c->ev1));
  *ms_out = ms / iters;
  API_END(c)
}
