/* A plain-C caller of the shading queries (include/trb.h): it compiles and links against libtrb with nothing but the header, pins
 * the layout of every query and result struct, prints every sizeof / offsetof, and prints the status of each entry point called
 * with null arguments (checked before any device is touched, so it runs without a GPU). */
#include <stddef.h>
#include <stdio.h>
#include "trb.h"

_Static_assert(sizeof(trb_bsdf_eval_query) == 32 && offsetof(trb_bsdf_eval_query, bxdf) == 12 && offsetof(trb_bsdf_eval_query, wi) == 16,
               "trb_bsdf_eval_query layout");
_Static_assert(sizeof(trb_bsdf_sample_query) == 32 && offsetof(trb_bsdf_sample_query, u) == 16 && offsetof(trb_bsdf_sample_query, u_comp) == 24,
               "trb_bsdf_sample_query layout");
_Static_assert(sizeof(trb_bsdf_sample_result) == 32 && offsetof(trb_bsdf_sample_result, pdf) == 12 && offsetof(trb_bsdf_sample_result, sampled) == 28,
               "trb_bsdf_sample_result layout");
_Static_assert(sizeof(trb_light_query) == 32 && offsetof(trb_light_query, time) == 12 && offsetof(trb_light_query, light) == 24,
               "trb_light_query layout");
_Static_assert(sizeof(trb_light_sample_result) == 80 && offsetof(trb_light_sample_result, delta) == 28 && offsetof(trb_light_sample_result, shadow) == 32,
               "trb_light_sample_result layout");
_Static_assert(sizeof(trb_light_pdf_query) == 32 && offsetof(trb_light_pdf_query, wi) == 16 && offsetof(trb_light_pdf_query, light) == 28,
               "trb_light_pdf_query layout");
_Static_assert(sizeof(trb_emit_query) == 32 && offsetof(trb_emit_query, n) == 16 && offsetof(trb_emit_query, inst) == 28, "trb_emit_query layout");
_Static_assert(TRB_BXDF_REFLECTION == 1 && TRB_BXDF_TRANSMISSION == 2 && TRB_BXDF_DIFFUSE == 4 && TRB_BXDF_GLOSSY == 8 && TRB_BXDF_SPECULAR == 16 &&
               TRB_BXDF_ALL == 31, "BxDFType bits");

#define S(T) printf(#T " sizeof %d\n", (int)sizeof(T))
#define F(T, f) printf(#T "." #f " %d\n", (int)offsetof(T, f))

int main(void) {
    S(trb_bsdf_eval_query); F(trb_bsdf_eval_query, wo); F(trb_bsdf_eval_query, bxdf); F(trb_bsdf_eval_query, wi); F(trb_bsdf_eval_query, pad);
    S(trb_bsdf_sample_query); F(trb_bsdf_sample_query, wo); F(trb_bsdf_sample_query, bxdf); F(trb_bsdf_sample_query, u);
    F(trb_bsdf_sample_query, u_comp); F(trb_bsdf_sample_query, pad);
    S(trb_bsdf_sample_result); F(trb_bsdf_sample_result, f); F(trb_bsdf_sample_result, pdf); F(trb_bsdf_sample_result, wi);
    F(trb_bsdf_sample_result, sampled);
    S(trb_light_query); F(trb_light_query, p); F(trb_light_query, time); F(trb_light_query, u); F(trb_light_query, light); F(trb_light_query, pad);
    S(trb_light_sample_result); F(trb_light_sample_result, li); F(trb_light_sample_result, pdf); F(trb_light_sample_result, wi);
    F(trb_light_sample_result, delta); F(trb_light_sample_result, shadow);
    S(trb_light_pdf_query); F(trb_light_pdf_query, p); F(trb_light_pdf_query, time); F(trb_light_pdf_query, wi); F(trb_light_pdf_query, light);
    S(trb_emit_query); F(trb_emit_query, w); F(trb_emit_query, time); F(trb_emit_query, n); F(trb_emit_query, inst);
    trb_intersection rec = {0};
    trb_bsdf_eval_query eq = {{0, 0, 1}, TRB_BXDF_ALL, {0, 0, 1}, 0};
    trb_bsdf_sample_query sq = {{0, 0, 1}, TRB_BXDF_ALL, {0.5f, 0.5f}, 0.5f, 0};
    trb_light_query lq = {{0, 0, 0}, 0.0f, {0.5f, 0.5f}, 0, 0};
    trb_light_pdf_query pq = {{0, 0, 0}, 0.0f, {0, 0, 1}, 0};
    trb_emit_query mq = {{0, 0, 1}, 0.0f, {0, 0, 1}, 0};
    float out4[4], pdf, rgb[3];
    trb_bsdf_sample_result bs;
    trb_light_sample_result ls;
    uint32_t lights[4];
    printf("status trb_bsdf_eval %d\n", (int)trb_bsdf_eval(NULL, 1, &rec, &eq, out4));
    printf("status trb_bsdf_eval_device %d\n", (int)trb_bsdf_eval_device(NULL, 1, &rec, &eq, out4, NULL));
    printf("status trb_bsdf_sample %d\n", (int)trb_bsdf_sample(NULL, 1, &rec, &sq, &bs));
    printf("status trb_bsdf_sample_device %d\n", (int)trb_bsdf_sample_device(NULL, 1, &rec, &sq, &bs, NULL));
    printf("status trb_light_sample %d\n", (int)trb_light_sample(NULL, 1, &lq, &ls));
    printf("status trb_light_sample_device %d\n", (int)trb_light_sample_device(NULL, 1, &lq, &ls, NULL));
    printf("status trb_light_pdf %d\n", (int)trb_light_pdf(NULL, 1, &pq, &pdf));
    printf("status trb_light_pdf_device %d\n", (int)trb_light_pdf_device(NULL, 1, &pq, &pdf, NULL));
    printf("status trb_emitted %d\n", (int)trb_emitted(NULL, 1, &mq, rgb));
    printf("status trb_emitted_device %d\n", (int)trb_emitted_device(NULL, 1, &mq, rgb, NULL));
    printf("status trb_scene_lights %d\n", (int)trb_scene_lights(NULL, lights));
    printf("status TRB_INVALID_ARG %d\n", (int)TRB_INVALID_ARG);
    return 0;
}
