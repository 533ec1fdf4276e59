// Prints the route nfi_route.h picks for each request read from stdin, one request per line:
//   fwd|bwd [key=value ...]
// keys: mode, S, fine, zfine, extra, A, normals, peers, view, ws (workspace bytes, 0 = no
// workspace), dbg (debug bits of mlp_mode), grads (backward: comma-separated gradient outputs).
// Output, one line per request: the route, "+normals" when render_normals_pipe follows, or
// "refused: <message>".
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "nfi_route.h"

static const char* route_name(nfi::Route r) {
  switch (r) {
    case nfi::Route::kPipe: return "pipe";
    case nfi::Route::kPipeVd: return "pipe_vd";
    case nfi::Route::kSimt: return "simt";
    case nfi::Route::kSimtVd: return "simt_vd";
    case nfi::Route::kWgradOneSweep: return "wgrad_planes";
    case nfi::Route::kPipeAndWgrad: return "pipe+wgrad";
    case nfi::Route::kWgrad: return "wgrad";
    case nfi::Route::kRefused: return "refused";
  }
  return "?";
}

static float g_dummy[1];

static bool set_grad(nfi_render_grads& g, const char* name) {
  struct {
    const char* name;
    float** slot;
  } outs[] = {{"planes", &g.grad_planes},   {"w1", &g.grad_w1},
              {"b1", &g.grad_b1},           {"w2", &g.grad_w2},
              {"b2", &g.grad_b2},           {"palette", &g.grad_palette},
              {"beta", &g.grad_beta},       {"alpha", &g.grad_alpha},
              {"origins", &g.grad_origins}, {"dirs", &g.grad_dirs},
              {"view", &g.grad_view_features}, {"w3", &g.grad_w3},
              {"b3", &g.grad_b3}};
  for (auto& o : outs)
    if (!strcmp(o.name, name)) {
      *o.slot = g_dummy;
      return true;
    }
  if (!strcmp(name, "extra")) {  // an upstream gradient of the extra output
    g.g_extra = g.out_extra = g_dummy;
    return true;
  }
  return false;
}

int main() {
  char line[1024];
  while (fgets(line, sizeof(line), stdin)) {
    nfi_render_params p;
    nfi_render_grads g;
    memset(&p, 0, sizeof(p));
    memset(&g, 0, sizeof(g));
    p.num_samples = 64;
    p.n_attention = 10;
    p.fine_sampling = 1;
    p.z_fine = g_dummy;
    p.workspace = g_dummy;
    p.workspace_bytes = NFI_BACKWARD_WORKSPACE_BYTES;
    g.g_rgb = g.out_rgb = g.out_mask = g_dummy;
    const bool bwd = !strncmp(line, "bwd", 3);
    if (!bwd && strncmp(line, "fwd", 3)) return 2;
    int dbg = 0;
    for (char* tok = strtok(line + 3, " \n"); tok; tok = strtok(nullptr, " \n")) {
      char* eq = strchr(tok, '=');
      if (!eq) return 2;
      *eq = 0;
      const char* v = eq + 1;
      const long n = strtol(v, nullptr, 0);
      if (!strcmp(tok, "mode")) p.mlp_mode = (int32_t)n;
      else if (!strcmp(tok, "S")) p.num_samples = (int32_t)n;
      else if (!strcmp(tok, "fine")) p.fine_sampling = (int32_t)n;
      else if (!strcmp(tok, "zfine")) p.z_fine = n ? g_dummy : nullptr;
      else if (!strcmp(tok, "extra")) p.extra_mode = (int32_t)n;
      else if (!strcmp(tok, "A")) p.n_attention = (int32_t)n;
      else if (!strcmp(tok, "normals")) p.use_sdf = p.compute_normals = (int32_t)n;
      else if (!strcmp(tok, "peers")) p.n_peers = (int32_t)n;
      else if (!strcmp(tok, "view")) p.view_features = n ? g_dummy : nullptr;
      else if (!strcmp(tok, "ws")) {
        p.workspace_bytes = (size_t)n;
        p.workspace = n ? g_dummy : nullptr;
      } else if (!strcmp(tok, "dbg")) dbg = (int)n;
      else if (!strcmp(tok, "grads")) {
        char* save = nullptr;
        for (char* name = strtok_r(eq + 1, ",", &save); name; name = strtok_r(nullptr, ",", &save))
          if (!set_grad(g, name)) return 2;
      } else {
        return 2;
      }
    }
    p.mlp_mode |= dbg;
    const nfi::Plan r = bwd ? nfi::route_backward(p, g) : nfi::route_forward(p);
    if (r.route == nfi::Route::kRefused)
      printf("refused: %s\n", r.refusal);
    else
      printf("%s%s\n", route_name(r.route), r.normals_pipe ? "+normals" : "");
  }
  return 0;
}
