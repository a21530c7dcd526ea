// plot_html.cpp — see plot_html.h.
#include "plot_html.h"

#include <math.h>
#include <stdio.h>

namespace glhtml {

std::string num(const char* fmt, double v) {
    if (isnan(v)) return "NaN";
    if (isinf(v)) return v > 0 ? "Infinity" : "-Infinity";
    char b[64];
    snprintf(b, sizeof b, fmt, v);
    return b;
}

std::string quote(const std::string& s) {
    std::string o = "\"";
    for (unsigned char c : s) {
        if (c == '"' || c == '\\') { o += '\\'; o += (char)c; }
        else if (c == '<') o += "\\u003c";                         // no "</script>" inside a script
        else if (c < 0x20) { char b[8]; snprintf(b, sizeof b, "\\u%04x", c); o += b; }
        else o += (char)c;
    }
    return o + "\"";
}

static std::string axis(const std::string& label, double lo = NAN, double hi = NAN) {
    const std::string ticks = isnan(lo) ? "" : ",\"ticks\":{\"min\":" + num("%g", lo) + ",\"max\":" + num("%g", hi) + "}";
    return "[{\"type\":\"linear\",\"scaleLabel\":{\"display\":true,\"fontSize\":16,\"labelString\":" + quote(label) + "}" + ticks + "}]";
}

std::string dataset_head(const Dataset& ds) {
    char col[48];
    snprintf(col, sizeof col, "\"rgba(%d,%d,%d,0.94)\"", ds.rgb[0], ds.rgb[1], ds.rgb[2]);
    std::string o = "{\"label\":" + quote(ds.label) + ",\"borderColor\":" + col + ",\"backgroundColor\":" + col + ",\"pointBackgroundColor\":" + col +
                    ",\"fill\":false";
    o += ds.line ? ",\"showLine\":true,\"pointRadius\":0,\"borderWidth\":" + num("%g", ds.width)
                 : ",\"showLine\":false,\"borderWidth\":0,\"pointRadius\":" + num("%g", ds.width);
    if (ds.stepped) o += ",\"steppedLine\":true";
    return o + ",\"pointHitRadius\":6,\"data\":[";
}

std::string chart_open(const Chart& c, int width, int height) {
    const std::string& n = c.name;
    char dims[64];
    snprintf(dims, sizeof dims, " width=\"%d\" height=\"%d\"", width, height);
    return "<canvas id=\"" + n + "\"" + dims + "></canvas>\n<script>\n/*chart " + n + " begin*/var cfg_" + n + " = {\"type\":\"line\",\"data\":{\"datasets\":[";
}

std::string chart_close(const Chart& c) {
    const std::string& n = c.name;
    return "]},\"options\":{\"responsive\":false,\"animation\":{\"duration\":0},\"legend\":{\"display\":" + std::string(c.legend ? "true" : "false") +
           "},\"tooltips\":{\"mode\":\"nearest\"},\"hover\":{\"mode\":\"nearest\"},\"scales\":{\"xAxes\":" + axis(c.xlabel) +
           ",\"yAxes\":" + axis(c.ylabel, c.ymin, c.ymax) + "}}};/*chart " + n + " end*/\n(function() {\n  var chart = new Chart(document.getElementById(\"" +
           n + "\"), cfg_" + n + ");\n" + c.tooltip_js + "\n  chart.update();\n})();\n</script>\n";
}

std::string chart_html(const Chart& c, int width, int height) {
    std::string cfg = chart_open(c, width, height);
    for (size_t d = 0; d < c.data.size(); d++) {
        const Dataset& ds = c.data[d];
        if (d) cfg += ",";
        cfg += dataset_head(ds);
        std::string pts;
        pts.reserve(ds.x.size() * 24);
        for (size_t i = 0; i < ds.x.size(); i++) {
            if (i) pts += ",";
            pts += "{\"x\":" + num(ds.xfmt, ds.x[i]) + ",\"y\":" + num(ds.yfmt, ds.y[i]) + "}";
        }
        cfg += pts + "]}";
    }
    return cfg + chart_close(c);
}

std::string page_open(const std::string& title) {
    return "<!DOCTYPE html>\n<html><head><meta charset=\"utf-8\"><title>" + title +
           "</title>\n<script src=\"https://code.jquery.com/jquery-2.2.4.min.js\"></script>\n"
           "<script src=\"https://cdnjs.cloudflare.com/ajax/libs/Chart.js/2.3.0/Chart.bundle.js\"></script>\n</head><body>\n";
}

const char* page_close() { return "</body></html>\n"; }

std::string page(const std::string& title, const std::string& body) { return page_open(title) + body + page_close(); }

}  // namespace glhtml
