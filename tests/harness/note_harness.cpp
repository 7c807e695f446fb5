// tests/harness/note_harness.cpp -- the note encryption and scanning core (note_core.cuh) compiled for the HOST, so tests
// can compare the exact code the kernels run with the spec (oracle/notes.py) without a GPU.  The fixed base is multiplied by
// plain double-and-add here (no window table).  Test-only.
#include "host_math.hpp"
#include "note_core.cuh"
#include <cstring>
using namespace og;

template <class F> static F load(const uint8_t* b) { uint32_t c[8]; memcpy(c, b, 32); return F::from_canonical(c); }
template <class F> static void store(uint8_t* b, const F& v) { uint32_t c[8]; v.to_canonical(c); memcpy(b, c, 32); }

static const Fr* constants() {
    static Fr c[MIMC_ROUNDS];
    static bool init = false;
    if (!init) { mimc7_round_constants(c); init = true; }
    return c;
}

extern "C" {
// base_xy: BASE as two canonical words
void nh_public_keys(const uint8_t* keys, uint64_t n, const uint8_t* base_xy, uint8_t* pk_x, uint8_t* pk_odd) {
    BjjBase base{load<Fr>(base_xy), load<Fr>(base_xy + 32), nullptr};
    for (uint64_t i = 0; i < n; i++) {
        Fr v = load<Fr>(keys + 32 * i), x, y;
        bjj_to_pub(&x, &y, &base, &v);
        store(pk_x + 32 * i, x);
        pk_odd[i] = fr_is_odd(y) ? 1 : 0;
    }
}

void nh_encrypt(const uint8_t* pk_x, const uint8_t* pk_odd, const uint8_t* nul, const uint8_t* sec, const uint8_t* tok,
                const uint64_t* amounts, const uint8_t* eph, uint64_t n, const uint8_t* base_xy, uint8_t* rec, uint8_t* cm,
                uint8_t* status) {
    const Fr* c = constants();
    BjjBase base{load<Fr>(base_xy), load<Fr>(base_xy + 32), nullptr};
    for (uint64_t i = 0; i < n; i++) {
        uint32_t a[8] = {(uint32_t)amounts[i], (uint32_t)(amounts[i] >> 32), 0, 0, 0, 0, 0, 0};
        Fr m[4] = {load<Fr>(nul + 32 * i), load<Fr>(sec + 32 * i), load<Fr>(tok + 32 * i), Fr::from_canonical(a)}, k;
        uint32_t w[NOTE_RECORD_WORDS];
        status[i] = note_encrypt_one(load<Fr>(pk_x + 32 * i), pk_odd[i] != 0, m, load<Fr>(eph + 32 * i), base,
                                     [&](int j) { return c[j]; }, w, &k);
        memcpy(rec + 160 * i, w, 160);
        store(cm + 32 * i, k);
    }
}

// keys: canonical and nonzero mod l (the caller's checks); window selects the variable-base multiplier
void nh_scan(const uint8_t* keys, uint32_t n_keys, const uint8_t* recs, const uint8_t* cms, uint64_t n, int window,
             uint32_t* owner, uint8_t* plain) {
    const Fr* c = constants();
    auto cf = [&](int j) { return c[j]; };
    for (uint64_t i = 0; i < n; i++) {
        uint32_t w[NOTE_RECORD_WORDS], cm[8];
        memcpy(w, recs + 160 * i, 160);
        memcpy(cm, cms + 32 * i, 32);
        memset(plain + 128 * i, 0, 128);
        Fr ex, ey;
        if (!note_prepare_one(w, cm, &ex, &ey)) { owner[i] = NOTE_MALFORMED; continue; }
        owner[i] = NOTE_NOT_OWNED;
        for (uint32_t j = 0; j < n_keys; j++) {
            uint32_t v[8];
            memcpy(v, keys + 32 * j, 32);
            Fr m[4];
            bool owned = window ? note_decrypt_one<true>(ex, ey, v, w, cm, cf, m) : note_decrypt_one<false>(ex, ey, v, w, cm, cf, m);
            if (owned) {
                owner[i] = j;
                for (int k = 0; k < 4; k++) store(plain + 128 * i + 32 * k, m[k]);
                break;
            }
        }
    }
}
}
