/*
 * b200hash_napi.c -- N-API (Node-API, C) addon exposing the GPU digests to the JS SDK of the reference.
 *
 * js/src/blob.ts:31-69 `blobUpload` does
 *     const contentMd5    = createHash("md5").update(data).digest("base64");
 *     const contentSha256 = createHash("sha256").update(data).digest("base64");
 * and then talks to the control plane / object store with its own gRPC client and fetch().  Only those two lines are
 * arithmetic, so that is what the addon replaces: `hashesMany(buffers)` hashes any number of Uint8Array payloads in ONE
 * GPU batch (b200blob_hashes_many -> b200h_hash_batch_host) and returns the base64 strings blobCreate wants;
 * `shouldUpload(n)` is createInput's 2 MiB gate.  The patched blob.ts is in INTEGRATION.md section 3.
 *
 * Build (on a machine with Node headers):  cc -shared -fPIC -I$(node -p "process.config.variables.node_prefix")/include/node \
 *     -Iinclude bindings/node/b200hash_napi.c -Lmodal_client_b200 -lb200hash -o b200hash.node
 * `node` is not installed in this image: tests/test_c_host.py compiles this file against tests/c/node_api.h, a small
 * stand-in for the Node-API subset used here, and drives it from C exactly as Node would.
 */
#include <node_api.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "b200blob.h"

static b200h_ctx* g_ctx = NULL;

static napi_value throw_error(napi_env env, const char* msg) {
    napi_throw_error(env, NULL, msg);
    return NULL;
}

static int ensure_context(napi_env env) {
    if (g_ctx) return 1;
    if (b200h_create(0, 0, 0, &g_ctx) != 0) { /* no CPU fallback: without an H100 the addon throws */
        throw_error(env, b200h_last_error(NULL));
        return 0;
    }
    return 1;
}

/* hashesMany(buffers: Uint8Array[]): { md5: string[], sha256: string[] } -- standard base64 with padding, as
 * createHash(...).digest("base64") returns (blob.ts:35-36). */
static napi_value HashesMany(napi_env env, napi_callback_info info) {
    size_t argc = 1;
    napi_value arg, result = NULL, md5_arr, sha_arr;
    bool is_array = false;
    uint32_t n = 0;
    if (napi_get_cb_info(env, info, &argc, &arg, NULL, NULL) != napi_ok || argc < 1) return throw_error(env, "hashesMany(buffers) expects one argument");
    if (napi_is_array(env, arg, &is_array) != napi_ok || !is_array) return throw_error(env, "hashesMany: argument must be an array of Uint8Array");
    if (!ensure_context(env)) return NULL;
    napi_get_array_length(env, arg, &n);
    const uint8_t** data = (const uint8_t**)calloc(n ? n : 1, sizeof *data);
    uint64_t* len = (uint64_t*)calloc(n ? n : 1, sizeof *len);
    char* md5 = (char*)malloc((size_t)(n ? n : 1) * B200BLOB_MD5_B64_LEN);
    char* sha = (char*)malloc((size_t)(n ? n : 1) * B200BLOB_SHA256_B64_LEN);
    char err[B200BLOB_ERR_MAX];
    if (!data || !len || !md5 || !sha) {
        throw_error(env, "out of memory");
        goto done;
    }
    for (uint32_t i = 0; i < n; ++i) {
        napi_value el;
        napi_typedarray_type type;
        size_t length = 0;
        void* ptr = NULL;
        if (napi_get_element(env, arg, i, &el) != napi_ok ||
            napi_get_typedarray_info(env, el, &type, &length, &ptr, NULL, NULL) != napi_ok || type != napi_uint8_array) {
            throw_error(env, "hashesMany: every element must be a Uint8Array");
            goto done;
        }
        data[i] = (const uint8_t*)ptr; /* the payload stays where V8 keeps it: the library gathers from these addresses */
        len[i] = (uint64_t)length;
    }
    if (n && b200blob_hashes_many(g_ctx, data, len, n, md5, sha, err) != 0) {
        throw_error(env, err);
        goto done;
    }
    napi_create_object(env, &result);
    napi_create_array_with_length(env, n, &md5_arr);
    napi_create_array_with_length(env, n, &sha_arr);
    for (uint32_t i = 0; i < n; ++i) {
        napi_value s;
        napi_create_string_utf8(env, md5 + (size_t)i * B200BLOB_MD5_B64_LEN, NAPI_AUTO_LENGTH, &s);
        napi_set_element(env, md5_arr, i, s);
        napi_create_string_utf8(env, sha + (size_t)i * B200BLOB_SHA256_B64_LEN, NAPI_AUTO_LENGTH, &s);
        napi_set_element(env, sha_arr, i, s);
    }
    napi_set_named_property(env, result, "md5", md5_arr);
    napi_set_named_property(env, result, "sha256", sha_arr);
done:
    free(data);
    free(len);
    free(md5);
    free(sha);
    return result;
}

/* shouldUpload(nbytes: number): boolean -- strictly more than 2 MiB (go/function.go:193, js createInput) */
static napi_value ShouldUpload(napi_env env, napi_callback_info info) {
    size_t argc = 1;
    napi_value arg, out;
    double nbytes = 0;
    if (napi_get_cb_info(env, info, &argc, &arg, NULL, NULL) != napi_ok || argc < 1 ||
        napi_get_value_double(env, arg, &nbytes) != napi_ok)
        return throw_error(env, "shouldUpload(nbytes) expects a number");
    napi_get_boolean(env, b200blob_should_upload(nbytes < 0 ? 0 : (uint64_t)nbytes) != 0, &out);
    return out;
}

NAPI_MODULE_INIT() {
    napi_value fn;
    napi_create_function(env, "hashesMany", NAPI_AUTO_LENGTH, HashesMany, NULL, &fn);
    napi_set_named_property(env, exports, "hashesMany", fn);
    napi_create_function(env, "shouldUpload", NAPI_AUTO_LENGTH, ShouldUpload, NULL, &fn);
    napi_set_named_property(env, exports, "shouldUpload", fn);
    return exports;
}
