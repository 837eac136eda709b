/* The AOV albedo of a BSDF (DESIGN.md §4 "AOVs") — TEST INFRASTRUCTURE, shared by the AOV oracles (oracle_aov/aov.cpp and
 * oracle_adaptive_aov/adaptive_aov.cpp). Include it after the oracle's shading code (BSDF, Lobe, Col): the sum over the BSDF's
 * lobes, in allocation order, of colour x the lobe's own Fresnel at cos 1 (diffuse lobes: colour; transmission lobes:
 * colour x (1 - F)); MERL: pi x BSDF::eval(n, n, all lobes); each channel clamped to [0, 1]. */
#pragma once

static Col aov_albedo(const BSDF& b) {
    Col acc(0.0f);
    for (int i = 0; i < b.n_lobes; ++i) {
        const Lobe& l = b.lobes[i];
        switch (l.kind) {
            case L_LAMBERT: case L_OREN_NAYAR: acc = acc + l.c; break;
            case L_SPEC_REFL: case L_TORRANCE_SPARROW: acc = acc + l.c * l.fresnel.eval(1.0f); break;
            case L_SPEC_TRANS: case L_MICROFACET_TRANS: acc = acc + l.c * (Col(1.0f) - l.fresnel.eval(1.0f)); break;
            case L_MERL: acc = b.eval(b.n, b.n, BX_ALL) * PI; break;
        }
    }
    return acc.clamp();
}
